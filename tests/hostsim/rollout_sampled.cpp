// rollout_sampled.cpp -- the device source of rollout_sampled_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/{per_env,space_sample}.cuh
// through tests/hostsim/cuda_shim.h and runs, for every CTA of the grid b200gym_rollout_sampled launches, what the
// kernel's CTA does: sample_stream_start, the ticket, rollout_sampled_env for each of its envs, and
// sample_stream_finish from the last CTA to arrive.  The batch layout and the reset / step entry points are those of
// rollout.cpp (included below), so tests/test_rollout_sampled_cpu.py can compare one sampled rollout with T kernel-A
// steps of the same batch.  The record lives in host memory here; the argument set-up copies b200gym_rollout_sampled.
#include "rollout.cpp"

struct longlong2 { long long x, y; };
static inline longlong2 make_longlong2(long long x, long long y) { longlong2 r = {x, y}; return r; }

#include "../../gym_b200/csrc/space_sample.cuh"

namespace {
constexpr int64_t kCta = 256;   // rollout_sampled_kernel's CTA (kThreads in b200gym.cu)
}

extern "C" {

// one b200gym_rollout_sampled launch of T steps on a host record (bgym::kSampleRecordWords words); override may be
// NULL, low / high are read for Box kinds -> the number of invalid actions met (-1: bad kind)
int64_t hs_ros_rollout(const Batch *B, uint64_t *record, const uint64_t *override_pcg64, int64_t n_choices, double low,
                       double high, int32_t T, void *actions_out, float *obs, double *reward, uint8_t *term,
                       uint8_t *trunc, float *final_obs, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    bgym::SampleStream s{};
    s.record = record;
    if (override_pcg64) {
        s.use_override = 1;
        for (int k = 0; k < 4; k++) s.override_words[k] = override_pcg64[k];
    }
    s.advance = bgym::lcg_jump_map((bgym::u128)((int64_t)T * B->n));
    const bgym::LcgMap hop = bgym::lcg_jump_map((bgym::u128)(B->n - 1));
    RolloutDraws d{hop.mult, hop.geo, n_choices > 0 ? (double)n_choices : low, n_choices > 0 ? 0.0 : high, 0};
    for (uint64_t last = (uint64_t)(B->n - 1); last != 0; last >>= 4) d.jump_digits++;
    const int64_t blocks = (B->n + kCta - 1) / kCta;
    const int64_t rc = dispatch(B->kind, n_choices > 0 ? B200GYM_ACT_I64 : B200GYM_ACT_F32, [&](auto k, auto *) -> int64_t {
        for (int64_t b = 0; b < blocks; b++) {
            const bgym::Pcg64 start = bgym::sample_stream_start(s);
            const bool last_cta = record[4]++ == (uint64_t)(blocks - 1);
            for (int64_t i = b * kCta; i < (b + 1) * kCta && i < B->n; i++)
                rollout_sampled_env<decltype(k)::value>(a, i, T, last_obs, d, start, bgym::kLcgJump);
            if (last_cta) bgym::sample_stream_finish(s, start);
        }
        return 0;
    });
    return rc < 0 ? rc : (int64_t)invalid;
}

}  // extern "C"
