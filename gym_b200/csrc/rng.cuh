// rng.cuh -- numpy's bit generator on the device.
//
// Every reference env owns Generator(PCG64(SeedSequence(seed)))
// (gym/utils/seeding.py:24-26; Env.reset re-seeds iff a seed is given,
// gym/core.py:149-151) and autoreset continues that private stream
// (gym/vector/sync_vector_env.py:154).  To give the same initial states as the
// reference for the same seed, each device env carries the same 256-bit PCG64
// record and the seeding kernel evaluates SeedSequence's hash on the device
// (numpy costs ~7 us/seed on the host: 7 s for 2^20 envs).
//
// HBM layout: one 32-byte record per env {state_hi, state_lo, inc_hi, inc_lo}
// (AoS on purpose: only the few lanes that reset in a step touch it, and a
// 32 B record is exactly one DRAM sector).
#pragma once
#include <cstdint>

namespace bgym {

typedef unsigned __int128 u128;

struct Pcg64 {
    u128 state;
    u128 inc;
};

__host__ __device__ __forceinline__ u128 make_u128(uint64_t hi, uint64_t lo) {
    return ((u128)hi << 64) | (u128)lo;
}

// PCG64 default multiplier 0x2360ED051FC65DA44385DF649FCCF645
__host__ __device__ __forceinline__ void pcg64_advance(Pcg64 &g) {
    const u128 mult = make_u128(0x2360ED051FC65DA4ULL, 0x4385DF649FCCF645ULL);
    g.state = g.state * mult + g.inc;
}

// pcg_setseq_128_srandom_r: how numpy's PCG64(SeedSequence) initialises
__host__ __device__ __forceinline__ void pcg64_seed(Pcg64 &g, u128 initstate, u128 initseq) {
    g.state = 0;
    g.inc = (initseq << 1) | 1;
    pcg64_advance(g);
    g.state += initstate;
    pcg64_advance(g);
}

// XSL-RR output of the *advanced* state
__host__ __device__ __forceinline__ uint64_t pcg64_next64(Pcg64 &g) {
    pcg64_advance(g);
    const uint64_t hi = (uint64_t)(g.state >> 64), lo = (uint64_t)g.state;
    const uint64_t x = hi ^ lo;
    const unsigned rot = (unsigned)(hi >> 58);
    return (x >> rot) | (x << ((64u - rot) & 63u));
}

// Generator.random(): 53 random bits scaled by 2^-53
__host__ __device__ __forceinline__ double pcg64_next_double(Pcg64 &g) {
    return (double)(pcg64_next64(g) >> 11) * (1.0 / 9007199254740992.0);
}

// Generator.uniform(low, high) = low + (high - low) * random()
// (two separately rounded operations -- the TU is built with -fmad=false)
__host__ __device__ __forceinline__ double pcg64_uniform(Pcg64 &g, double low, double high) {
    const double range = high - low;
    return low + range * pcg64_next_double(g);
}

// ---- jump-ahead: the state `delta` draws later, in O(log delta) ----
// `delta` steps of the LCG are the affine map state -> mult * state + geo * inc, where mult = A^delta and
// geo = A^(delta-1) + ... + A + 1 (mod 2^128) do not depend on inc.
struct LcgMap {
    u128 mult;
    u128 geo;
};

// `first`, then `second`
__host__ __device__ constexpr LcgMap lcg_compose(LcgMap first, LcgMap second) {
    return {second.mult * first.mult, second.mult * first.geo + second.geo};
}

// pcg_advance_lcg_128 (PCG's square-and-multiply over the bits of delta) with inc = 1
__host__ __device__ constexpr LcgMap lcg_jump_map(u128 delta) {
    u128 cur_mult = ((u128)0x2360ED051FC65DA4ULL << 64) | (u128)0x4385DF649FCCF645ULL, cur_plus = 1;
    u128 acc_mult = 1, acc_plus = 0;
    while (delta > 0) {
        if (delta & 1) {
            acc_mult *= cur_mult;
            acc_plus = acc_plus * cur_mult + cur_plus;
        }
        cur_plus = (cur_mult + 1) * cur_plus;
        cur_mult *= cur_mult;
        delta >>= 1;
    }
    return {acc_mult, acc_plus};
}

__host__ __device__ __forceinline__ void pcg64_apply(Pcg64 &g, const LcgMap &m) {
    g.state = m.mult * g.state + m.geo * g.inc;
}

// numpy's PCG64.advance(delta) on the state words (the buffered 32-bit draw is not numpy's to clear here)
__host__ __device__ inline void pcg64_jump(Pcg64 &g, u128 delta) { pcg64_apply(g, lcg_jump_map(delta)); }

// The jump a sampling thread makes to the start of its elements, one table entry per non-zero hex digit of delta:
// m[k][d] is the map of d * 16^k steps.  8 KB, built by the compiler, read-only in global memory.
struct LcgJumpTable {
    LcgMap m[16][16];
};

__host__ __device__ constexpr LcgJumpTable make_lcg_jump_table() {
    LcgJumpTable t{};
    for (int k = 0; k < 16; k++) {
        const LcgMap unit = k == 0 ? lcg_jump_map(1) : lcg_compose(t.m[k - 1][15], t.m[k - 1][1]);
        t.m[k][0] = LcgMap{1, 0};
        t.m[k][1] = unit;
        for (int d = 2; d < 16; d++) t.m[k][d] = lcg_compose(t.m[k][d - 1], unit);
    }
    return t;
}

static __device__ const LcgJumpTable kLcgJump = make_lcg_jump_table();

// pcg64_jump for a 64-bit delta through a copy of kLcgJump (the kernels stage the rows they use in shared memory):
// 2 multiplies per non-zero hex digit instead of ~3 per bit
__host__ __device__ __forceinline__ void pcg64_jump_table(Pcg64 &g, uint64_t delta, const LcgJumpTable &table) {
    for (int k = 0; delta != 0; k++, delta >>= 4)
        if (delta & 15) pcg64_apply(g, table.m[k][delta & 15]);
}

// ---- one element of a batched action space's sample(): one 64-bit draw each, in C order ----
// MultiDiscrete.sample: (random(shape) * nvec).astype(int64) (gym/spaces/multi_discrete.py:123); the cast rounds
// toward zero
__host__ __device__ __forceinline__ long long sample_multidiscrete(Pcg64 &g, double n) {
    return (long long)(pcg64_next_double(g) * n);
}

// Box.sample of a bounded float Box: uniform(low, high).astype(float32) (gym/spaces/box.py:171-222); low and high
// are the float32 bounds widened to float64, the cast rounds to nearest
__host__ __device__ __forceinline__ float sample_box(Pcg64 &g, double low, double high) {
    return (float)pcg64_uniform(g, low, high);
}

// SeedSequence(seed).generate_state(4, uint64) for a seed given as four
// little-endian uint32 entropy words (seed < 2^128; shorter seeds are
// zero-padded, which hashes identically to numpy's own padding).
__host__ __device__ inline void seed_sequence_4x64(const uint32_t ent[4], uint64_t out[4]) {
    const uint32_t INIT_A = 0x43b0d7e5u, MULT_A = 0x931e8875u;
    const uint32_t INIT_B = 0x8b51f9ddu, MULT_B = 0x58f38dedu;
    const uint32_t MIX_L = 0xca01f9ddu, MIX_R = 0x4973f715u;
    uint32_t hc = INIT_A;
    uint32_t pool[4];
    auto hashmix = [&hc, MULT_A](uint32_t v) {
        v ^= hc;
        hc *= MULT_A;
        v *= hc;
        v ^= v >> 16;
        return v;
    };
#pragma unroll
    for (int i = 0; i < 4; i++) pool[i] = hashmix(ent[i]);
#pragma unroll
    for (int src = 0; src < 4; src++) {
#pragma unroll
        for (int dst = 0; dst < 4; dst++) {
            if (src != dst) {
                const uint32_t h = hashmix(pool[src]);
                uint32_t r = MIX_L * pool[dst] - MIX_R * h;
                r ^= r >> 16;
                pool[dst] = r;
            }
        }
    }
    uint32_t o[8];
    hc = INIT_B;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint32_t v = pool[i & 3];
        v ^= hc;
        hc *= MULT_B;
        v *= hc;
        v ^= v >> 16;
        o[i] = v;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) out[k] = (uint64_t)o[2 * k] | ((uint64_t)o[2 * k + 1] << 32);
}

__host__ __device__ inline void pcg64_from_entropy(Pcg64 &g, const uint32_t ent[4]) {
    uint64_t w[4];
    seed_sequence_4x64(ent, w);
    pcg64_seed(g, make_u128(w[0], w[1]), make_u128(w[2], w[3]));
}

// 32-byte HBM record <-> registers
__device__ __forceinline__ Pcg64 pcg64_load(const uint64_t *rec) {
    const ulonglong2 a = reinterpret_cast<const ulonglong2 *>(rec)[0];
    const ulonglong2 b = reinterpret_cast<const ulonglong2 *>(rec)[1];
    Pcg64 g;
    g.state = make_u128(a.x, a.y);
    g.inc = make_u128(b.x, b.y);
    return g;
}

__device__ __forceinline__ void pcg64_store(uint64_t *rec, const Pcg64 &g) {
    // inc never changes after seeding: only the state half is written back
    reinterpret_cast<ulonglong2 *>(rec)[0] =
        make_ulonglong2((uint64_t)(g.state >> 64), (uint64_t)g.state);
}

__device__ __forceinline__ void pcg64_store_full(uint64_t *rec, const Pcg64 &g) {
    reinterpret_cast<ulonglong2 *>(rec)[0] =
        make_ulonglong2((uint64_t)(g.state >> 64), (uint64_t)g.state);
    reinterpret_cast<ulonglong2 *>(rec)[1] =
        make_ulonglong2((uint64_t)(g.inc >> 64), (uint64_t)g.inc);
}

}  // namespace bgym
