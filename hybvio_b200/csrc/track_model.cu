// hybvio_b200/csrc/track_model.cu -- hv_track_model_kernel: triangulation + prepareVisualUpdate of a batch of tracks on the
// device (one CTA per track; body and algorithm notes in track_model.cuh). Replaces, for the EKF's visual updates, the host
// sequence extractCameraPoseTrail -> Triangulator::triangulate -> prepareVisualUpdate of src/odometry/backend.cpp:1050-1160.
#include "track_model.cuh"
#include "hv_device_once.cuh"
#include <stdlib.h>

__global__ void __launch_bounds__(TM_NT, 2) hv_track_model_kernel(TmArgs a)
{
    extern __shared__ __align__(16) double tm_dyn[];
    tm_body(a, tm_dyn, blockIdx.x);
}

// Group launch (hv_ekf_group_visual_tracks): CTA i runs the chain step args[i] of one filter of the group (blocks in device memory)
__global__ void __launch_bounds__(TM_NT, 2) hv_track_model_group_kernel(const TmArgs* __restrict__ args)
{
    extern __shared__ __align__(16) double tm_dyn[];
    tm_group_body(args, blockIdx.x, tm_dyn);
}

cudaError_t tm_launch(const TmArgs& a, cudaStream_t s)
{
    static bool seen[64];                             // per device (hv_common.cuh)
    if (hv_first_use_on_device(seen)) {
        cudaError_t e = cudaFuncSetAttribute(hv_track_model_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tm_smem_bytes());
        if (e != cudaSuccess) return e;
    }
    static const bool pdlAllowed = getenv("HV_EKF_NO_PDL") == nullptr;
    if (a.pdl && pdlAllowed) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(a.ntracks); cfg.blockDim = dim3(TM_NT); cfg.dynamicSmemBytes = tm_smem_bytes(); cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        return cudaLaunchKernelEx(&cfg, hv_track_model_kernel, a);
    }
    TmArgs b = a;
    b.pdl = 0;
    hv_track_model_kernel<<<a.ntracks, TM_NT, tm_smem_bytes(), s>>>(b);
    return cudaGetLastError();
}

cudaError_t tm_launch_group(const TmArgs* hArgs, const TmArgs* dArgs, int count, cudaStream_t s)
{
    static bool seen[64];
    if (hv_first_use_on_device(seen)) {
        cudaError_t e = cudaFuncSetAttribute(hv_track_model_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tm_smem_bytes());
        if (e != cudaSuccess) return e;
    }
    // the blocks' pdl words are already in device memory: without the launch attribute the kernel's griddepcontrol instructions
    // find the previous grid complete and return at once
    static const bool pdlAllowed = getenv("HV_EKF_NO_PDL") == nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(count); cfg.blockDim = dim3(TM_NT); cfg.dynamicSmemBytes = tm_smem_bytes(); cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = hArgs[0].pdl && pdlAllowed ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, hv_track_model_group_kernel, dArgs);
}
