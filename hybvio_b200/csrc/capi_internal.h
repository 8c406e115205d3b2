// hybvio_b200/csrc/capi_internal.h -- host-side objects behind the opaque C handles.
#pragma once
#include "hv_common.cuh"
#include "../../include/hybvio_b200.h"
#include <vector>
#include <string>

#define HV_TABLE_CAPACITY 1024   // pyramids per context
#define HV_EKF_STAGES 4          // pinned staging blocks of hv_ekf_group_run_device per context (calls the host may run ahead)

void hv_set_error(const char* fmt, ...);
#define HV_CUDA(call)                                                                           \
    do {                                                                                        \
        cudaError_t e_ = (call);                                                                \
        if (e_ != cudaSuccess) {                                                                \
            hv_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return e_ == cudaErrorMemoryAllocation ? HV_ERR_OOM : HV_ERR_CUDA;                  \
        }                                                                                       \
    } while (0)

struct hv_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool ownStream = false;
    HvPyrDesc* d_table = nullptr;
    std::vector<int> freeSlots;
    long long launches = 0;
    // Staging of the host-buffer calls (LK, the detectors, the two-view geometry): one pinned block + one device block, grown on demand
    void* h_stage = nullptr; void* d_stage = nullptr; size_t stageBytes = 0;
    void* hd_stage = nullptr;          // device alias of h_stage (mapped pinned memory): results are written straight to the host
    // Device scratch of the detectors and the two-view geometry (capi.cu: ctx_scratch), only ever grown. Every call carves its own regions
    // from the start of it, so calls share it: all their launches are on `stream`, and a call's regions are dead once its last launch has run.
    void* d_scratch = nullptr; size_t scratchBytes = 0;
    unsigned* d_done = nullptr;        // completion counter of the polled launches (device)
    unsigned doneCount = 0, seq = 0;   // host mirror of the counter / sequence number of the last polled launch
    // EKF group staging (hv_ekf_group_run_device): a call's argument blocks reach the device in one copy out of a ring of pinned blocks
    // (block i is refilled once the copy out of it has completed, evEkfStage[i]) into one device block
    void* h_ekfStage[HV_EKF_STAGES] = {}; size_t h_ekfStageBytes[HV_EKF_STAGES] = {}; cudaEvent_t evEkfStage[HV_EKF_STAGES] = {};
    int ekfStageNext = 0;
    void* d_ekfStage = nullptr; size_t ekfStageBytes = 0;
    // Side stream for work that the main stream need not wait for (created on first use; ekf_capi.cu: outlier checks of a device-resident
    // op list). hv_ctx_sync waits for both.
    cudaStream_t sideStream = nullptr;
    cudaStream_t covStream = nullptr;   // full launch of an IMU burst whose mean part went ahead (ekf_capi.cu: predict_launch)
};

struct hv_pyr {
    hv_ctx* ctx = nullptr;
    int slot = -1;
    int w = 0, h = 0, win = 0, nlevels = 0;
    void* d_mem = nullptr;
    size_t bytes = 0;
    HvPyrDesc desc;
};

int hv_ctx_reserve_stage(hv_ctx* ctx, size_t bytes);
// Spins until done() holds (a condition on mapped pinned memory that a kernel on `stream` writes); checks the stream for errors,
// and for a kernel that finished without signalling, every 4096 spins.
template <class Done> int hv_poll(cudaStream_t stream, const char* who, Done done)
{
    for (unsigned long long spins = 1;; spins++) {
        if (done()) break;
        if ((spins & 0xfff) == 0) {
            const cudaError_t q = cudaStreamQuery(stream);
            if (q == cudaErrorNotReady) continue;
            if (q != cudaSuccess) { hv_set_error("%s: %s while waiting for the result", who, cudaGetErrorString(q)); return HV_ERR_CUDA; }
            if (done()) break;
            hv_set_error("%s: the kernel finished without signalling its completion", who); return HV_ERR_STATE;
        }
    }
    __atomic_thread_fence(__ATOMIC_ACQUIRE);
    return HV_OK;
}

// kernels (pyramid.cu, lk.cu)
cudaError_t hv_launch_pyr_fused(const HvPyrDesc* table, const unsigned short* idx, const uint8_t* const* src, const int* srcPitch,
                                const uint8_t* const* level0, const int* level0Pitch, const int* nlevels,
                                int n, int w0, int h0, int maxNlevels, cudaStream_t stream);
