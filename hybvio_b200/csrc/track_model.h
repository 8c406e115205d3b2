// hybvio_b200/csrc/track_model.h -- arguments of the per-track measurement-model kernel (track_model.cuh / track_model.cu),
// shared by the kernel, its launcher and the C ABI (ekf_capi.cu: hv_ekf_track_models).
#pragma once
#include <stddef.h>

#define TM_NT 256
#define TM_MAXPOSE 21                         // cameraTrailLength 20 + the current pose
#define TM_MAXOBS (2 * TM_MAXPOSE)
#define TM_MAXCOL (7 * TM_MAXOBS + 1)
#define TM_MAXN (20 + 7 * (TM_MAXPOSE - 1))
#define TM_POS 0
#define TM_ORI 6
#define TM_SFT 19
#define TM_CAM 20

enum { TM_OK = 0, TM_HYBRID, TM_BEHIND, TM_BAD_COND, TM_NO_CONVERGENCE, TM_BAD_DEPTH, TM_UNKNOWN_PROBLEM };   // TriangulatorStatus, output.hpp:21-29
enum { TM_VU_OK = 0, TM_VU_ZERO_DEPTH = 1, TM_VU_BEHIND = 2, TM_VU_NOT_RUN = -1 };
#define TM_SKIPPED (-1)                        // triangulation not attempted: the chain already has its successful updates (backend.cpp:1240-1247)                              // PrepareVuStatus, output.hpp:15-19

struct TmArgs {
    const double* m;            // state mean (device), N entries
    int N, stereo, timeShift, ntracks;
    double Rc[2][9];            // imuToCamera / secondImuToCamera rotation, row-major
    double base[2][3];          // their translation ("baseline" of CameraPose)
    unsigned gnIterations;      // odometry.triangulationGaussNewtonIterations
    double convThreshold, convR, rcondThreshold, minDist, maxDist;
    const int* npose;           // [ntracks]
    const int* idx;             // [ntracks][TM_MAXPOSE]   poseTrailIndex: 0 = current pose, k = trail slot k - 1
    const double* ip;           // [ntracks][TM_MAXOBS][2] normalised image points: camera 0 poses, then camera 1 poses
    const double* vel;          // [ntracks][TM_MAXOBS][2] their velocities
    int* status;                // [ntracks][4]  TriangulatorStatus, PrepareVuStatus, rows, cols
    double* pf;                 // [ntracks][4]  triangulated point, depth
    double* dpf;                // [ntracks][3 (7 TM_MAXPOSE + 1)] d pf / d (poses, t) after the stereo sum (column-major), or NULL
    double* H;                  // [ntracks][Hstride]  rows x cols column-major, ld = rows
    double* f;                  // [ntracks][2 TM_MAXOBS]
    size_t Hstride;
    int trackOffset;            // CTA b handles track b + trackOffset (chains launch one track at a time out of a packed batch)
    int counterMax;             // with counter != NULL: skip (status TM_SKIPPED) once *counter >= counterMax
    const int* counter;         // successful updates so far in a chain issued without host round trips (hv_ekf_visual_tracks)
    int pdl, padPdl;            // chain link: launched with programmatic stream serialisation (starts while the previous kernel of the
                                // stream drains, waits in griddepcontrol.wait before it reads anything that kernel wrote)
};

#ifdef __CUDACC__
#include <cuda_runtime.h>
cudaError_t tm_launch(const TmArgs& a, cudaStream_t s);      // grid = a.ntracks CTAs of TM_NT threads
// Group launch (hv_ekf_group_visual_tracks): CTA i runs track dArgs[i].trackOffset of dArgs[i], a block in device memory; hArgs is the
// host copy of the same blocks (hArgs[0].pdl: the launch follows a kernel of the chains on the stream)
cudaError_t tm_launch_group(const TmArgs* hArgs, const TmArgs* dArgs, int count, cudaStream_t s);
#endif
