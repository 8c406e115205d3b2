// tests/emu/cuda_emu_atomics.h -- what the Shi-Tomasi kernels (good_features.cu) need on top of cuda_emu.h and cuda_emu_ballot.h: integer
// and max atomics, integer warp shuffles, the warp max reduction and a few bit / rounding intrinsics. Test infrastructure only; include
// after cuda_emu_ballot.h.
#pragma once
#include "cuda_emu_ballot.h"

inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicMax(unsigned* p, unsigned v)
{
    unsigned old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
// full-warp collectives on integers: EVERY lane of the warp must call them
inline long long emu_warp_exchange(long long v, int src)
{
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* slot = emu::cta->xch.data() + (size_t)w * 32;
    memcpy(&slot[lane], &v, sizeof(v));
    emu::cta->wbar[w]->arrive_and_wait();
    long long r;
    memcpy(&r, &slot[src & 31], sizeof(r));
    emu::cta->wbar[w]->arrive_and_wait();
    return r;
}
inline int __shfl_sync(unsigned, int v, int src) { return (int)emu_warp_exchange(v, src); }
inline int __shfl_up_sync(unsigned, int v, int delta)
{
    const int lane = threadIdx.x & 31;
    const int r = (int)emu_warp_exchange(v, lane >= delta ? lane - delta : lane);
    return lane >= delta ? r : v;
}
inline unsigned __reduce_max_sync(unsigned, unsigned v)
{
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* slot = emu::cta->xch.data() + (size_t)w * 32;
    slot[lane] = (double)v;
    emu::cta->wbar[w]->arrive_and_wait();
    unsigned m = 0u;
    for (int i = 0; i < 32; i++) m = (unsigned)slot[i] > m ? (unsigned)slot[i] : m;
    emu::cta->wbar[w]->arrive_and_wait();
    return m;
}
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, sizeof(f)); return f; }
inline float __double2float_rn(double d) { volatile float f = (float)d; return f; }
inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
inline float2 make_float2(float x, float y) { return float2{x, y}; }
