// rollout_from_mlp.cpp -- the per-branch driver of rollout_from_mlp_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose configuration struct and kind dispatch it shares) and runs
// rollout_from_mlp_env for every branch.  tests/test_rollout_from_mlp_cpu.py compares it with the MLP rollout drivers
// run on a batch restored from the same rows.  The argument set-up copies b200gym_rollout_from_mlp: no handle arrays,
// a.n = B, each branch's flag byte in storage of its own, the statistics staged as the kernel stages them (mean null:
// raw inputs), and a shared policy read where the kernel reads its shared-memory copy.
#include "rollout.cpp"

extern "C" {

// one b200gym_rollout_from_mlp launch of T steps over nb branches (h2 = 0: one hidden layer; act: a
// b200gym_mlp_activation; noise NULL: none); B supplies the configuration only.  end_rows / end_obs NULL: no end
// states.  *bad is set to 1 if a row index was out of range -> the number of invalid actions met (-1: bad kind)
int64_t hs_rfm_rollout_from_mlp(const Batch *B, const unsigned char *rows, int64_t n_rows, const int64_t *row_idx,
                                int64_t nb, const float *params, int per_branch, int h1, int h2, int act, int32_t T,
                                const float *noise, const double *mean, const double *var, double eps, float clip,
                                double *returns, int32_t *lengths, uint8_t *ended, void *first, unsigned char *end_rows,
                                float *end_obs, unsigned long long *bad) {
    unsigned long long invalid = 0, seen = 0;
    std::vector<uint8_t> flags((size_t)nb);
    StepArgs a = args_of(*B, &invalid, &seen, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    a.state = nullptr; a.elapsed = nullptr; a.rng = nullptr;
    a.flags = flags.data();
    a.n = nb; a.count = nb;
    double sd[24];
    const int64_t rc = dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR ||
                                         B->kind == B200GYM_ACROBOT ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                                [&](auto k, auto *) -> int64_t {
                                    constexpr int KIND = decltype(k)::value, R = B200GYM_MLP_RELU,
                                                  H = B200GYM_MLP_TANH;
                                    constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
                                    if (mean)
                                        for (int c = 0; c < D; c++) sd[c] = norm_sd(var[c], eps);
                                    const int64_t P = mlp_param_count<K, D>(h1, h2);
                                    const bool vec = h1 % 4 == 0 && (!per_branch || P % 4 == 0);
                                    const RolloutFromMlpArgs p{
                                        {rows, n_rows, row_idx, returns, lengths, ended, end_rows, end_obs, bad},
                                        {params, per_branch ? P : 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr},
                                        noise,
                                        first};
                                    for (int64_t b = 0; b < nb; b++) {
                                        const float *w = params + b * p.mlp.stride;
                                        auto run = [&](auto st, auto gl, auto ac) {
                                            rollout_from_mlp_env<KIND, decltype(st)::value, decltype(gl)::value,
                                                                 decltype(ac)::value>(a, b, b, T, w, p, mean, sd, clip);
                                        };
                                        using T1 = std::true_type;
                                        using F0 = std::false_type;
                                        using AR = std::integral_constant<int, R>;
                                        using AH = std::integral_constant<int, H>;
                                        const bool s = end_rows != nullptr, g = per_branch != 0;
                                        if (act == H) {
                                            if (s) g ? run(T1{}, T1{}, AH{}) : run(T1{}, F0{}, AH{});
                                            else g ? run(F0{}, T1{}, AH{}) : run(F0{}, F0{}, AH{});
                                        } else {
                                            if (s) g ? run(T1{}, T1{}, AR{}) : run(T1{}, F0{}, AR{});
                                            else g ? run(F0{}, T1{}, AR{}) : run(F0{}, F0{}, AR{});
                                        }
                                    }
                                    return 0;
                                });
    return rc < 0 ? rc : (int64_t)invalid;
}

}  // extern "C"
