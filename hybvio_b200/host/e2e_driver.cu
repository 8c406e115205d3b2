// hybvio_b200/host/e2e_driver.cu -- native caller of the C ABI for bench.py's `e2e` number.
//
// Plays the role of the reference's Session::process (src/odometry/backend.cpp:716-867) for one stereo frame after the
// other, entirely through the public host-buffer entry points of include/hybvio_b200.h -- the calls the C++ adapters in
// this directory make -- so that the end-to-end measurement contains the ABI, the host<->device copies and every
// synchronisation, but not the Python interpreter of the harness. Not part of the product library
// (libhv_e2e_driver.so links libhybvio_b200.so).
#include "../../include/hybvio_b200.h"
#include <cuda_runtime.h>
#include <chrono>
#include <vector>

extern "C" {

typedef struct hv_e2e_frame {
    const uint8_t* left; const uint8_t* right;   // host (pinned) gray images; right == NULL: mono (BASELINE config 1)
    size_t stride;
    const float* init_xy;                        // predicted end points for the temporal LK call (n x 2)
    const hv_ekf_op* ops;                        // the frame's EKF calls, HOST pointers (predicts, checks/updates, symmetrise, augment)
    int nops;
} hv_e2e_frame;

// pyr[0..1] = previous left/right, pyr[2..3] = scratch for the current frame (swapped every frame).
// pose_out: 20 doubles (inertial state after the last frame). elapsed_ms: device time of the whole loop (CUDA events
// on the tracker stream, taken after both streams are idle).
//
// host_phase_us (optional, 4 doubles): host wall time summed over the frames of {pyramid submit, temporal LK, stereo LK,
// EKF op list} -- where the end-to-end time goes (the calls are synchronous, so host time == critical path).
static int e2e_run(hv_ctx* trk, hv_ctx* ekf_ctx, hv_pyr** pyr, hv_ekf* ekf, const float* points, int n, const hv_e2e_frame* frames,
                   int nframes, double* pose_out, float* elapsed_ms, double* host_phase_us)
{
    using clk = std::chrono::steady_clock;
    auto us = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
    double ph[4] = {0, 0, 0, 0};
    std::vector<float> nxt(2 * (size_t)n), nxt2(2 * (size_t)n);
    std::vector<uint8_t> st(n);
    std::vector<int32_t> ts(n);
    std::vector<int> vu(64);
    std::vector<double> chi2(64), m(hv_ekf_state_dim(ekf));
    hv_pyr* p[4] = {pyr[0], pyr[1], pyr[2], pyr[3]};
    cudaStream_t s = (cudaStream_t)hv_ctx_stream(trk);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    hv_ctx_sync(trk); hv_ctx_sync(ekf_ctx);
    cudaEventRecord(e0, s);
    int rc = HV_OK;
    // Frame k+1 is handed to the tracker as soon as frame k's optical flow is done (the reference creates the
    // tracker::Image on the frame-input thread, src/api/api.cpp:602-605): its H2D copy and pyramid build run on the tracker
    // stream while the EKF stream works on frame k. The pyramids of frame k-1 are free at that point and take frame k+1.
    auto submit = [&](int k, hv_pyr* const* dst) {
        const uint8_t* img[2] = {frames[k].left, frames[k].right};
        const size_t strides[2] = {frames[k].stride, frames[k].stride};
        return hv_pyr_build_batch(dst, img, strides, frames[k].right ? 2 : 1, 0);           // H2D + one kernel, asynchronous
    };
    {
        const auto t0 = clk::now();
        hv_pyr* cur[2] = {p[2], p[3]};
        if (nframes > 0) rc = submit(0, cur);
        ph[0] += us(t0, clk::now());
    }
    for (int k = 0; k < nframes && rc == HV_OK; k++) {
        const hv_e2e_frame& f = frames[k];
        hv_pyr* cur[2] = {p[2], p[3]};
        for (int i = 0; i < 2 * n; i++) nxt[i] = f.init_xy[i];
        // the IMU samples that arrived before the frame (backend.cpp:716-760 processes them first): queued and launched without waiting,
        // so that the state propagation runs beside the optical flow
        int nimu = 0;
        while (nimu < f.nops && f.ops[nimu].kind != HV_EKF_OP_VISUAL) nimu++;
        const auto t0i = clk::now();
        if (nimu > 0) rc = hv_ekf_run_host(ekf, f.ops, nimu, nullptr, nullptr, nullptr);
        if (rc == HV_OK) rc = hv_ekf_flush(ekf);
        if (rc != HV_OK) break;
        const auto t1 = clk::now();
        rc = hv_lk_track(trk, p[0], cur[0], points, nxt.data(), st.data(), ts.data(), n, 1, 20, 0.03, 1e-3);   // sync
        if (rc != HV_OK) break;
        const auto t2 = clk::now();
        if (f.right) rc = hv_lk_track(trk, cur[0], cur[1], nxt.data(), nxt2.data(), st.data(), ts.data(), n, 0, 20, 0.03, 1e-3);
        if (rc != HV_OK) break;
        const auto t3 = clk::now();
        if (k + 1 < nframes) { hv_pyr* nxtp[2] = {p[0], p[1]}; rc = submit(k + 1, nxtp); if (rc != HV_OK) break; }
        const auto t3b = clk::now();
        if ((int)vu.size() < f.nops) { vu.resize(f.nops); chi2.resize(f.nops); }
        rc = hv_ekf_run_host(ekf, f.ops + nimu, f.nops - nimu, vu.data(), chi2.data(), m.data());    // one synchronisation for the frame's measurements
        const auto t4 = clk::now();
        ph[0] += us(t3, t3b); ph[1] += us(t1, t2); ph[2] += us(t2, t3); ph[3] += us(t3b, t4) + us(t0i, t1);
        hv_pyr* q0 = p[0]; hv_pyr* q1 = p[1]; p[0] = p[2]; p[1] = p[3]; p[2] = q0; p[3] = q1;
    }
    hv_ctx_sync(ekf_ctx);
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(elapsed_ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    for (int i = 0; i < 4; i++) pyr[i] = p[i];
    if (pose_out) for (int i = 0; i < 20; i++) pose_out[i] = m[i];
    if (host_phase_us) for (int i = 0; i < 4; i++) host_phase_us[i] = ph[i];
    return rc;
}

// ---- device-resident loop (bench.py's `value`): the same frame as above with every input already in HBM and no host
// synchronisation. Dependencies (LK(k) after the mean propagation of frame k: the flow predictor reads the propagated pose and the pose
// trail, src/odometry/backend.cpp:547-600 via src/tracker/tracker.cpp:59-63; visual updates(k) after LK(k); next propagation after the
// augmentation) are stream order on ONE stream; what does not depend on them runs beside it. A native caller keeps the launch rate
// independent of the Python interpreter of the harness.
typedef struct hv_dev_frame {
    const uint8_t* left; const uint8_t* right;   // device gray images
    size_t stride;
    const float* d_init_xy;                      // device: predicted end points (n x 2)
    const hv_ekf_op* ops;                        // the frame's EKF calls with DEVICE pointers; the first nimu ops are the IMU burst
    int nops, nimu;
} hv_dev_frame;

int hv_dev_run(hv_ctx* trk, hv_ctx* ekf_ctx, hv_pyr** pyr, hv_ekf* ekf, const float* d_points, float* d_next, float* d_next2,
               uint8_t* d_status, int32_t* d_ts, int n, const hv_dev_frame* frames, int nframes, float* elapsed_ms)
{
    // Stream sa (the tracker context's): pyramid builds only. Stream sb (the filter context's): the WHOLE dependent chain of a frame --
    // mean propagation -> optical flow (hv_lk_track_device_on_stream) -> visual updates -> the augmentation's mean -- so that no step of it
    // waits for a cross-stream event that has not fired long ago. Beside it, on streams of the library: the covariance part of the IMU
    // burst, and the outlier checks that precede the augmentation together with the augmentation's covariance.
    hv_pyr* p[4] = {pyr[0], pyr[1], pyr[2], pyr[3]};
    cudaStream_t sa = (cudaStream_t)hv_ctx_stream(trk), sb = (cudaStream_t)hv_ctx_stream(ekf_ctx);
    cudaEvent_t e0, e1, evPyr, evLk;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventCreateWithFlags(&evPyr, cudaEventDisableTiming); cudaEventCreateWithFlags(&evLk, cudaEventDisableTiming);
    hv_ctx_sync(trk); hv_ctx_sync(ekf_ctx);
    double* d_mean = nullptr;
    if (cudaMalloc(&d_mean, 20 * sizeof(double)) != cudaSuccess) {
        cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(evLk); cudaEventDestroy(evPyr);
        return HV_ERR_OOM;
    }
    cudaEventRecord(e0, sb);
    cudaEventRecord(evLk, sb);
    int rc = HV_OK, lastOps = 0;
    for (int k = 0; k < nframes && rc == HV_OK; k++) {
        const hv_dev_frame& f = frames[k];
        hv_pyr* cur[2] = {p[2], p[3]};
        const uint8_t* img[2] = {f.left, f.right};
        const size_t strides[2] = {f.stride, f.stride};
        cudaStreamWaitEvent(sa, evLk, 0);                                      // the pyramids about to be rebuilt were read by the previous frame's optical flow
        rc = hv_pyr_build_batch(cur, img, strides, f.right ? 2 : 1, 1);          // A: depends on nothing else
        if (rc != HV_OK) break;
        cudaEventRecord(evPyr, sa);
        rc = hv_ekf_run_device(ekf, f.ops, f.nimu);                            // B: IMU burst (queued) ...
        if (rc == HV_OK) rc = hv_ekf_predicted_mean_device(ekf, d_mean);       // ... its mean part first: all the flow predictor reads ...
        if (rc == HV_OK) rc = hv_ekf_flush(ekf);                               // ... the full launch (covariance) on the library's own stream
        if (rc != HV_OK) break;
        cudaStreamWaitEvent(sb, evPyr, 0);                                     // issued a whole frame of filter work ago: has fired
        // (f.d_init_xy: the predictor's output, read where it is)
        rc = hv_lk_track_device_on_stream(trk, sb, p[0], cur[0], d_points, f.d_init_xy, d_next, d_status, d_ts, n, 20, 0.03, 1e-3);
        if (rc == HV_OK && f.right) rc = hv_lk_track_device_on_stream(trk, sb, cur[0], cur[1], d_next, nullptr, d_next2, d_status, d_ts, n, 20, 0.03, 1e-3);
        if (rc != HV_OK) break;
        cudaEventRecord(evLk, sb);
        rc = hv_ekf_run_device(ekf, f.ops + f.nimu, f.nops - f.nimu);         // joins the covariance launch, then the visual updates
        if (rc == HV_OK) rc = hv_ekf_flush(ekf);
        lastOps = f.nops - f.nimu;
        hv_pyr* q0 = p[0]; hv_pyr* q1 = p[1]; p[0] = p[2]; p[1] = p[3]; p[2] = q0; p[3] = q1;
    }
    // the last frame's decisions come back to the host (this also waits for the outlier checks the library issued on its side stream)
    if (rc == HV_OK && lastOps > 0) { std::vector<int> vu(lastOps); std::vector<double> chi2(lastOps); rc = hv_ekf_run_device_results(ekf, lastOps, vu.data(), chi2.data()); }
    cudaStreamWaitEvent(sb, evPyr, 0);
    cudaEventRecord(e1, sb);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(elapsed_ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(evLk); cudaEventDestroy(evPyr);
    cudaFree(d_mean);
    for (int i = 0; i < 4; i++) pyr[i] = p[i];
    return rc;
}

int hv_e2e_run(hv_ctx* trk, hv_ctx* ekf_ctx, hv_pyr** pyr, hv_ekf* ekf, const float* points, int n, const hv_e2e_frame* frames,
               int nframes, double* pose_out, float* elapsed_ms)
{
    return e2e_run(trk, ekf_ctx, pyr, ekf, points, n, frames, nframes, pose_out, elapsed_ms, nullptr);
}

int hv_e2e_run_phases(hv_ctx* trk, hv_ctx* ekf_ctx, hv_pyr** pyr, hv_ekf* ekf, const float* points, int n, const hv_e2e_frame* frames,
                      int nframes, double* pose_out, float* elapsed_ms, double* host_phase_us)
{
    return e2e_run(trk, ekf_ctx, pyr, ekf, points, n, frames, nframes, pose_out, elapsed_ms, host_phase_us);
}
}
