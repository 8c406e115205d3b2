// hybvio_b200/csrc/ingest.cu -- frame ingest (SURVEY.md 8(f) N4): what tracker::Image::Factory does to a camera frame before the tracker
// sees it (src/tracker/image.cpp:274-308), on the device, writing straight into level 0 of the frame's pyramid:
//   colour -> gray   accelerated-arrays pixelwiseAffine({0.299, 0.587, 0.114 (, 0)}) on UFIXED8 images (image.cpp:360-366;
//                    AA/cpu/operations.cpp:145-177 pixelwiseAffineUnary<FixedPoint<uint8_t>>, AA/fixed_point.hpp:16-36)
//   undistort / rectify   UndistorterImplementation::undistort, CPU branch (src/tracker/undistorter.cpp:77-118): per output pixel
//                    pixelToRay (rectified camera) -> rayToPixel (original camera), bilinear interpolation in fp32, int(out + 0.5)
// The camera mapping of a session is fixed, so the adapter (hybvio_b200/host/cuda_undistorter.cpp) evaluates it ONCE per camera with the
// reference's own Camera classes (double precision) and hands the kernel a table: per output pixel floor(x), floor(y) and the two fp32
// fractions exactly as undistorter.cpp:93-94 forms them -- the kernel then only interpolates, in the reference's operation order, and is
// bit-exact for every camera model. Both kernels are streaming (one read, one write per pixel) and HBM / L2-bandwidth bound.
#include "hv_common.cuh"

// gray = T(sum_j coeff[j] * float(in[j])), v accumulated in fp32 from 0 in channel order (separate multiply and add), float(in) =
// (float)(value / 255.0) [lut], T(v) = (uint8)(255.0 * clamp(v, 0, 1) + 0.5) in double. p: the pixel's first channel.
__device__ __forceinline__ uint8_t hv_gray_pixel(const uint8_t* p, int channels, float c0, float c1, float c2, float c3, const float* lut)
{
    float v = 0.0f;
    v = __fadd_rn(v, __fmul_rn(c0, lut[p[0]]));
    if (channels > 1) v = __fadd_rn(v, __fmul_rn(c1, lut[p[1]]));
    if (channels > 2) v = __fadd_rn(v, __fmul_rn(c2, lut[p[2]]));
    if (channels > 3) v = __fadd_rn(v, __fmul_rn(c3, lut[p[3]]));
    double d = (double)v;
    d = d < 0.0 ? 0.0 : d > 1.0 ? 1.0 : d;
    return (uint8_t)(255.0 * d + 0.5);
}

__device__ __forceinline__ void hv_gray_lut(float* lut)
{
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = (float)((double)i / 255.0);
    __syncthreads();
}

__global__ void __launch_bounds__(256) hv_gray_kernel(const uint8_t* __restrict__ src, int srcPitch, int channels, int w, int h,
                                                      float c0, float c1, float c2, float c3, uint8_t* __restrict__ dst, int dstPitch)
{
    __shared__ float lut[256];
    hv_gray_lut(lut);
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    dst[(size_t)y * dstPitch + x] = hv_gray_pixel(src + (size_t)y * srcPitch + (size_t)x * channels, channels, c0, c1, c2, c3, lut);
}

// out(x, y) = int(sum over the 2 x 2 taps of in(y0 + iy, x0 + ix) * wx * wy + 0.5), taps in the order (0,0), (0,1), (1,0), (1,1) with
// wx = ix ? xfrac : 1 - xfrac; entries with x0 == HV_REMAP_INVALID give 0 (outside the source image / behind the camera).
// tap(row, col) returns in(row, col) as a float; it is called with col up to w and row up to h (see the readers below).
template <class Tap>
__device__ __forceinline__ uint8_t hv_remap_pixel(const HvRemapEntry& e, Tap tap)
{
    float out = 0.0f;
    if (e.x0 != HV_REMAP_INVALID) {
#pragma unroll
        for (int iy = 0; iy < 2; iy++) {
            const float wy = iy ? e.yfrac : __fsub_rn(1.0f, e.yfrac);
#pragma unroll
            for (int ix = 0; ix < 2; ix++) {
                const float wx = ix ? e.xfrac : __fsub_rn(1.0f, e.xfrac);
                out = __fadd_rn(out, __fmul_rn(__fmul_rn(tap(e.y0 + iy, e.x0 + ix), wx), wy));
            }
        }
    }
    return (uint8_t)(int)((double)out + 0.5);
}

// The reference reads a tap to the right of the last column / below the last row from whatever follows in memory (cv::Mat::at without a
// bounds check, undistorter.cpp:101): here such a tap reads the linear address too, clamped to the last byte of the image.
__device__ __forceinline__ float hv_remap_tap(const uint8_t* __restrict__ src, int srcPitch, int w, int h, int row, int col)
{
    const long long last = (long long)(h - 1) * srcPitch + (w - 1);
    long long a = (long long)row * srcPitch + col;
    a = a > last ? last : a;
    return (float)src[a];
}

__global__ void __launch_bounds__(256) hv_remap_kernel(const uint8_t* __restrict__ src, int srcPitch, int w, int h, const HvRemapEntry* __restrict__ table,
                                                       uint8_t* __restrict__ dst, int dstPitch)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const HvRemapEntry e = table[(size_t)y * w + x];
    dst[(size_t)y * dstPitch + x] = hv_remap_pixel(e, [&](int row, int col) { return hv_remap_tap(src, srcPitch, w, h, row, col); });
}

// Many frames in one launch (hv_ingest_frames): CTA b of the flattened grid belongs to job j = hv_batch_job(first, b) and covers 256
// pixels of one row. Each job runs one of three modes, uniform per CTA: colour only (gray into level 0), remap only (taps from the source at
// its own pitch, as hv_remap_kernel reads the staged frame) and colour + remap fused. The two-launch path writes gray into an intermediate
// of pitch w and remaps from it; the fused tap clamps the same linear index a = row * w + col to w * h - 1 and computes the gray value of
// pixel (a / w, a % w) from the colour source instead. Gray is a function of one pixel, so the bits are those of the two launches.
__global__ void __launch_bounds__(256) hv_ingest_batch_kernel(const __grid_constant__ IngestBatchArgs b)
{
    __shared__ float lut[256];
    const int g = blockIdx.x, j = hv_batch_job(b.first, g);
    const IngestJob& J = b.job[j];
    const int bx = (J.w + 255) >> 8, r = g - b.first[j], y = r / bx, x = (r - y * bx) * 256 + threadIdx.x;
    const int channels = J.channels;
    const float c0 = J.coeff[0], c1 = J.coeff[1], c2 = J.coeff[2], c3 = J.coeff[3];
    if (channels > 1) hv_gray_lut(lut);                                 // uniform per CTA
    if (x >= J.w) return;
    const uint8_t* __restrict__ src = J.src;
    const int pitch = J.srcPitch, w = J.w, h = J.h;
    uint8_t v;
    if (!J.table) {
        v = hv_gray_pixel(src + (size_t)y * pitch + (size_t)x * channels, channels, c0, c1, c2, c3, lut);
    } else {
        const HvRemapEntry e = J.table[(size_t)y * w + x];
        if (channels == 1) {
            v = hv_remap_pixel(e, [&](int row, int col) { return hv_remap_tap(src, pitch, w, h, row, col); });
        } else {
            const long long last = (long long)w * h - 1;
            v = hv_remap_pixel(e, [&](int row, int col) {
                long long a = (long long)row * w + col;
                a = a > last ? last : a;
                const int ar = (int)(a / w), ac = (int)(a - (long long)ar * w);
                return (float)hv_gray_pixel(src + (size_t)ar * pitch + (size_t)ac * channels, channels, c0, c1, c2, c3, lut);
            });
        }
    }
    J.dst[(size_t)y * J.dstPitch + x] = v;
}

cudaError_t hv_launch_gray(const uint8_t* src, int srcPitch, int channels, int w, int h, const float coeff[4], uint8_t* dst, int dstPitch, cudaStream_t s)
{
    hv_gray_kernel<<<dim3((w + 255) / 256, h), 256, 0, s>>>(src, srcPitch, channels, w, h, coeff[0], coeff[1], coeff[2], coeff[3], dst, dstPitch);
    return cudaGetLastError();
}
cudaError_t hv_launch_remap(const uint8_t* src, int srcPitch, int w, int h, const HvRemapEntry* table, uint8_t* dst, int dstPitch, cudaStream_t s)
{
    hv_remap_kernel<<<dim3((w + 255) / 256, h), 256, 0, s>>>(src, srcPitch, w, h, table, dst, dstPitch);
    return cudaGetLastError();
}
cudaError_t hv_launch_ingest_batch(const IngestBatchArgs& b, int njobs, cudaStream_t s)
{
    const int ctas = b.first[njobs];
    if (ctas <= 0) return cudaSuccess;
    hv_ingest_batch_kernel<<<ctas, 256, 0, s>>>(b);
    return cudaGetLastError();
}
