// cuda_shim.h -- just enough of the CUDA C++ dialect to compile gym_b200/csrc/{rng,envs,b2lite,lunar,walker,per_env}.cuh
// with a host compiler.  TEST INFRASTRUCTURE: tests/hostsim builds the device source for the CPU so that the
// `-m "not gpu"` suite can run the very code the kernels run, per-env drivers included, against the C oracle (see
// hostsim.cpp).  The host build is single-threaded: one lane, one warp.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#define __device__
#define __host__
#define __global__
#define __constant__
#define __forceinline__ inline
#define __noinline__

static inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline double __longlong_as_double(long long v) { double d; std::memcpy(&d, &v, 8); return d; }
static inline long long __double_as_longlong(double d) { long long v; std::memcpy(&v, &d, 8); return v; }

struct ulonglong2 { unsigned long long x, y; };
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { ulonglong2 r = {x, y}; return r; }
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
static inline float2 make_float2(float x, float y) { float2 r = {x, y}; return r; }
static inline float4 make_float4(float x, float y, float z, float w) { float4 r = {x, y, z, w}; return r; }

template <typename T>
static inline T __ldg(const T *p) { return *p; }
template <typename T>
static inline T atomicAdd(T *p, T v) { const T old = *p; *p = old + v; return old; }

// warp votes of a one-lane "warp"
static inline int __any_sync(unsigned, int p) { return p; }
static inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
static inline void __syncwarp(unsigned = 0xffffffffu) {}
