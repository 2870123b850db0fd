// sample_stream.cpp -- the device source of space_sample_stream_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/{rng,space_sample}.cuh
// through tests/hostsim/cuda_shim.h and runs, for every CTA of the grid b200gym_sample_space_stream launches, what the
// kernel's CTA does: sample_stream_start, the ticket, sample_stream_finish from the last CTA to arrive, and
// sample_thread with the hop derived from the start's inc.  tests/test_sample_stream_cpu.py compares consecutive calls
// with numpy's Generator.  The record lives in host memory here; the argument set-up copies b200gym_sample_space_stream.
#include "cuda_shim.h"

// the one vector type space_sample.cuh stores that the shim does not declare
struct longlong2 { long long x, y; };
static inline longlong2 make_longlong2(long long x, long long y) { longlong2 r = {x, y}; return r; }

#include "../../gym_b200/csrc/rng.cuh"
#include "../../gym_b200/csrc/space_sample.cuh"

extern "C" {

// one b200gym_sample_space_stream call on a host record (bgym::kSampleRecordWords words); override may be NULL
void hs_sample_space_stream(uint64_t *record, const uint64_t *override_pcg64, int64_t rows, int cols, int64_t n_choices,
                            const double *low, const double *high, void *out) {
    bgym::SampleArgs a{};
    a.total = rows * cols;
    a.cols = cols;
    a.n_choices = (double)n_choices;
    for (int c = 0; n_choices == 0 && c < cols; c++) { a.low[c] = low[c]; a.high[c] = high[c]; }
    bgym::SampleStream s{};
    s.record = record;
    if (override_pcg64) {
        s.use_override = 1;
        for (int k = 0; k < 4; k++) s.override_words[k] = override_pcg64[k];
    }
    s.advance = bgym::lcg_jump_map((bgym::u128)a.total);
    const int vec = n_choices > 0 ? 2 : 4;
    const int64_t blocks = bgym::sample_blocks(a.total, vec);
    const int64_t threads = blocks * bgym::kSampleThreads;
    bgym::sample_setup(a, threads, vec);
    for (int64_t b = 0; b < blocks; b++) {
        const bgym::Pcg64 start = bgym::sample_stream_start(s);
        if (record[4]++ == (uint64_t)(blocks - 1)) bgym::sample_stream_finish(s, start);
        for (int64_t t = b * bgym::kSampleThreads; t < (b + 1) * bgym::kSampleThreads; t++) {
            if (n_choices > 0)
                bgym::sample_thread<long long>(a, start, a.hop_geo * start.inc, (long long *)out, t, threads, bgym::kLcgJump);
            else
                bgym::sample_thread<float>(a, start, a.hop_geo * start.inc, (float *)out, t, threads, bgym::kLcgJump);
        }
    }
}

}  // extern "C"
