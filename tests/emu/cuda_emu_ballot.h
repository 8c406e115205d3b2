// tests/emu/cuda_emu_ballot.h -- the warp and block collectives the corner selection kernel (gftt_select.cu) needs on top of the host
// emulator of cuda_emu.h: warp ballot, block-wide OR, ffs and float bit reinterpretation. Test infrastructure only; include after cuda_emu.h.
#pragma once
#include "cuda_emu.h"
#include <atomic>

// full-warp ballot: EVERY lane of the warp must call it (as every kernel written for the emulator does)
inline unsigned __ballot_sync(unsigned, int p)
{
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* slot = emu::cta->xch.data() + (size_t)w * 32;
    slot[lane] = p ? 1.0 : 0.0;
    emu::cta->wbar[w]->arrive_and_wait();
    unsigned r = 0;
    for (int i = 0; i < 32; i++) if (slot[i] != 0.0) r |= 1u << i;
    emu::cta->wbar[w]->arrive_and_wait();
    return r;
}
inline std::atomic<int> emu_syncthreads_or_acc{0};
inline int __syncthreads_or(int p)
{
    emu::cta->bar.arrive_and_wait();               // every thread has read the result of the previous call
    if (threadIdx.x == 0) emu_syncthreads_or_acc = 0;
    emu::cta->bar.arrive_and_wait();
    if (p) emu_syncthreads_or_acc.fetch_or(1);
    emu::cta->bar.arrive_and_wait();
    return emu_syncthreads_or_acc.load();
}
inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, sizeof(u)); return u; }
