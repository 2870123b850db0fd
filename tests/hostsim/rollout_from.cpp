// rollout_from.cpp -- the per-branch driver of rollout_from_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose configuration struct and kind dispatch it shares) and runs
// rollout_from_env for every branch.  tests/test_rollout_from_cpu.py compares it with rollout_kernel's driver run on a
// batch restored from the same rows.  The argument set-up copies b200gym_rollout_from: no handle arrays, a.n = B, and
// each branch's flag byte in storage of its own (here a B-byte array indexed by the branch).
#include "rollout.cpp"

extern "C" {

// one b200gym_rollout_from launch of T steps over nb branches; B supplies the configuration only (kind, max_steps,
// autoreset, param0).  end_rows / end_obs NULL: no end states.  *bad is set to 1 if a row index was out of range
// -> the number of invalid actions met (-1: bad kind)
int64_t hs_rf_rollout_from(const Batch *B, const unsigned char *rows, int64_t n_rows, const int64_t *row_idx,
                           int64_t nb, const void *actions, int32_t T, double *returns, int32_t *lengths,
                           uint8_t *ended, unsigned char *end_rows, float *end_obs, unsigned long long *bad) {
    unsigned long long invalid = 0, seen = 0;
    std::vector<uint8_t> flags((size_t)nb);
    StepArgs a = args_of(*B, &invalid, &seen, actions, nullptr, nullptr, nullptr, nullptr, nullptr);
    a.state = nullptr; a.elapsed = nullptr; a.rng = nullptr;
    a.flags = flags.data();
    a.n = nb; a.count = nb;
    const RolloutFromArgs p{rows, n_rows, row_idx, returns, lengths, ended, end_rows, end_obs, bad};
    const int64_t rc = dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR ||
                                         B->kind == B200GYM_ACROBOT ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                                [&](auto k, auto *tag) -> int64_t {
                                    constexpr int KIND = decltype(k)::value;
                                    using ActT = std::remove_pointer_t<decltype(tag)>;
                                    for (int64_t b = 0; b < nb; b++) {
                                        if (end_rows) rollout_from_env<KIND, ActT, true>(a, b, b, T, p);
                                        else rollout_from_env<KIND, ActT, false>(a, b, b, T, p);
                                    }
                                    return 0;
                                });
    return rc < 0 ? rc : (int64_t)invalid;
}

// classic_row_bytes<KIND>() of the batch's kind (-1: bad kind)
int64_t hs_rf_row_bytes(const Batch *B) {
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t { return classic_row_bytes<decltype(k)::value>(); });
}

}  // extern "C"
