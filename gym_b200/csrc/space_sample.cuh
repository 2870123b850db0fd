// space_sample.cuh -- `envs.action_space.sample()` of a batched action space, one thread's share.
//
// gym/spaces/multi_discrete.py:123 and gym/spaces/box.py:171-222: both batched kinds of the in-scope ids take one
// 64-bit draw of the space's PCG64 stream per element, in C order, so element k of the flat [rows * cols] output is a
// function of draw k alone and the batch is produced in parallel (space_sample_kernel in b200gym.cu; the host build
// in tests/hostsim/sample_space.cpp runs sample_thread for every thread of the same grid in a plain loop).
//   layout: per round a thread writes one 16-byte vector of VEC consecutive elements (2 int64 / 4 float32), so a
//     warp's store is 512 contiguous bytes; the rounds are grid-strided.
//   jump: a thread reaches its first vector with pcg64_jump_table (2 multiplies per non-zero hex digit of the offset:
//     ~5 digits at 2^20 elements) and each next one with ONE multiply-add by the map of the grid stride, computed once
//     on the host.  sample_blocks sizes the grid for ~kSampleRounds rounds per thread, so the jumps cost well under
//     one multiply per element next to the one of each draw.  The kernel first stages the rows of the table its
//     offsets use in shared memory: the digits then cost one round trip to memory instead of one each.
#pragma once
#include <algorithm>
#include <cstdint>
#include <type_traits>

#include "rng.cuh"

namespace bgym {

constexpr int kSampleMaxCols = 32;
constexpr int kSampleRounds = 8;
constexpr int kSampleThreads = 256;

struct SampleArgs {
    Pcg64 start;                 // the generator before draw 0
    u128 hop_mult, hop_plus;     // state -> hop_mult * state + hop_plus: from after a thread's vector to its next one
    int64_t total;               // rows * cols
    int jump_digits;             // hex digits of the largest first-vector offset: the rows of kLcgJump in use
    int cols;
    double n_choices;            // MultiDiscrete: the n of every element (Box: unused)
    double low[kSampleMaxCols], high[kSampleMaxCols];   // Box: the bounds of each column, float32 widened to float64
};

// CTAs of kSampleThreads for `total` elements of VEC-element vectors: ~kSampleRounds vectors per thread, but never
// fewer CTAs than two per SM of an H100 (132 SMs) while there is a vector for each of their threads
__host__ inline int64_t sample_blocks(int64_t total, int vec) {
    const int64_t vectors = (total + vec - 1) / vec;
    const int64_t full = (vectors + kSampleThreads - 1) / kSampleThreads;   // one vector per thread
    return std::min<int64_t>(std::max<int64_t>((full + kSampleRounds - 1) / kSampleRounds, std::min<int64_t>(full, 264)),
                             INT32_MAX);
}

// the grid-stride map of a grid of `threads` threads, and the rows of kLcgJump its first jumps use
__host__ inline void sample_setup(SampleArgs &a, int64_t threads, int vec) {
    const LcgMap hop = lcg_jump_map((u128)(threads - 1) * (u128)vec);
    a.hop_mult = hop.mult;
    a.hop_plus = hop.geo * a.start.inc;
    a.jump_digits = 0;
    for (uint64_t last = (uint64_t)(threads - 1) * (uint64_t)vec; last != 0; last >>= 4) a.jump_digits++;
}

__host__ __device__ __forceinline__ void store_vec(long long *p, const long long (&v)[2]) {
    *reinterpret_cast<longlong2 *>(p) = make_longlong2(v[0], v[1]);
}
__host__ __device__ __forceinline__ void store_vec(float *p, const float (&v)[4]) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

// the elements of thread `thread` of a grid of `threads` threads: T = long long (MultiDiscrete) or float (Box)
template <typename T>
__host__ __device__ __forceinline__ void sample_thread(const SampleArgs &a, T *out, int64_t thread, int64_t threads,
                                                      const LcgJumpTable &table) {
    constexpr int VEC = 16 / sizeof(T);
    constexpr bool kDiscrete = std::is_same<T, long long>::value;
    const int64_t stride = threads * VEC;
    int64_t k0 = thread * VEC;
    if (k0 >= a.total) return;
    Pcg64 g = a.start;
    pcg64_jump_table(g, (uint64_t)k0, table);
    for (;;) {
        T v[VEC];
        int col = (kDiscrete || VEC % a.cols == 0) ? 0 : (int)(k0 % a.cols);
#pragma unroll
        for (int j = 0; j < VEC; j++) {
            if constexpr (kDiscrete) {
                v[j] = sample_multidiscrete(g, a.n_choices);
            } else {
                v[j] = sample_box(g, a.low[col], a.high[col]);
                col = col + 1 == a.cols ? 0 : col + 1;
            }
        }
        if (k0 + VEC <= a.total) {
            store_vec(out + k0, v);
        } else {   // the ragged last vector (draws past the end only move this thread's private copy)
#pragma unroll
            for (int j = 0; j < VEC; j++)
                if (k0 + j < a.total) out[k0 + j] = v[j];
        }
        k0 += stride;
        if (k0 >= a.total) break;
        g.state = a.hop_mult * g.state + a.hop_plus;
    }
}

}  // namespace bgym
