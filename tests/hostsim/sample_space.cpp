// sample_space.cpp -- the device source of space_sample_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/{rng,space_sample}.cuh
// through tests/hostsim/cuda_shim.h and runs sample_thread -- the kernel's own per-thread code -- for every thread of the
// grid b200gym_sample_space launches, in a plain loop.  tests/test_sample_actions_cpu.py compares it bit for bit with
// numpy's `action_space.sample()`, so the `-m "not gpu"` suite runs the jump table, the grid-stride hop, the
// per-element samplers and the thread-to-element mapping of the kernel.  What it does not run: the shared-memory
// staging of the table and nvcc's code generation -- that is what tests/test_gpu_sample_actions.py is for.
#include "cuda_shim.h"

// the one vector type space_sample.cuh stores that the shim does not declare
struct longlong2 { long long x, y; };
static inline longlong2 make_longlong2(long long x, long long y) { longlong2 r = {x, y}; return r; }

#include "../../gym_b200/csrc/rng.cuh"
#include "../../gym_b200/csrc/space_sample.cuh"

extern "C" {

// space_sample_kernel over the grid b200gym_sample_space launches (blocks = 0) or over `blocks` CTAs: sample_thread of
// every thread in turn.  Same arguments as b200gym_sample_space, out in host memory.
void hs_sample_space(const uint64_t pcg64[4], int64_t rows, int cols, int64_t n_choices, const double *low,
                     const double *high, void *out, int64_t blocks) {
    bgym::SampleArgs a{};
    a.start.state = bgym::make_u128(pcg64[0], pcg64[1]);
    a.start.inc = bgym::make_u128(pcg64[2], pcg64[3]);
    a.total = rows * cols;
    a.cols = cols;
    a.n_choices = (double)n_choices;
    for (int c = 0; n_choices == 0 && c < cols; c++) { a.low[c] = low[c]; a.high[c] = high[c]; }
    const int vec = n_choices > 0 ? 2 : 4;
    if (blocks <= 0) blocks = bgym::sample_blocks(a.total, vec);
    const int64_t threads = blocks * bgym::kSampleThreads;
    bgym::sample_setup(a, threads, vec);
    for (int64_t t = 0; t < threads; t++) {
        if (n_choices > 0) bgym::sample_thread<long long>(a, (long long *)out, t, threads, bgym::kLcgJump);
        else bgym::sample_thread<float>(a, (float *)out, t, threads, bgym::kLcgJump);
    }
}

// pcg64_jump (square-and-multiply) and pcg64_jump_table (the kernel's table walk) on {state_hi, state_lo, inc_hi, inc_lo}
void hs_pcg64_jump(uint64_t w[4], uint64_t delta_hi, uint64_t delta_lo, int table) {
    bgym::Pcg64 g{bgym::make_u128(w[0], w[1]), bgym::make_u128(w[2], w[3])};
    if (table) bgym::pcg64_jump_table(g, delta_lo, bgym::kLcgJump);
    else bgym::pcg64_jump(g, bgym::make_u128(delta_hi, delta_lo));
    w[0] = (uint64_t)(g.state >> 64);
    w[1] = (uint64_t)g.state;
}

}  // extern "C"
