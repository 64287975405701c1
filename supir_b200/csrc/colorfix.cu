// supir_b200 — SURVEY.md §8(f)1: colour fix applied to the decoded image inside the measured region
// (SUPIR/utils/colorfix.py: wavelet_blur :73-92, wavelet_decomposition :94-106, wavelet_reconstruction :108-120,
// calc_mean_std / adaptive_instance_normalization :45-71). fp32 NCHW planes, HBM-bound.
#include "common.cuh"
#include "supir_b200.h"

namespace supir {

// One level of the a-trous wavelet: low = blur_r(img) (3x3 kernel [1 2 1]^T[1 2 1]/16, dilation r, replicate padding);
// high (+)= img - low. `img` and `low` must be different buffers.
__global__ void wavelet_level_kernel(const float* __restrict__ img, float* __restrict__ low, float* __restrict__ high,
                                     int planes, int H, int W, int r, int accumulate) {
    const long long total = (long long)planes * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const int y = (int)((i / W) % H);
        const float* pl = img + (i / ((long long)W * H)) * H * W;
        const int y0 = max(y - r, 0), y2 = min(y + r, H - 1), x0 = max(x - r, 0), x2 = min(x + r, W - 1);
        const float c = pl[(long long)y * W + x];
        float acc = 0.0625f * pl[(long long)y0 * W + x0];
        acc = fmaf(0.125f, pl[(long long)y0 * W + x], acc);
        acc = fmaf(0.0625f, pl[(long long)y0 * W + x2], acc);
        acc = fmaf(0.125f, pl[(long long)y * W + x0], acc);
        acc = fmaf(0.25f, c, acc);
        acc = fmaf(0.125f, pl[(long long)y * W + x2], acc);
        acc = fmaf(0.0625f, pl[(long long)y2 * W + x0], acc);
        acc = fmaf(0.125f, pl[(long long)y2 * W + x], acc);
        acc = fmaf(0.0625f, pl[(long long)y2 * W + x2], acc);
        low[i] = acc;
        if (high) high[i] = (accumulate ? high[i] : 0.f) + (c - acc);
    }
}

// per-plane sum and sum of squares (fp64), deterministic: per-block partials + last-block ticket
__global__ void plane_stats_kernel(const float* __restrict__ x, long long hw, double* __restrict__ ws, int planes) {
    __shared__ double sh[2][32];
    __shared__ int is_last;
    const int p = blockIdx.y, nblk = gridDim.x;
    double* sums = ws;
    double* partial = ws + 2LL * planes;
    unsigned int* tickets = reinterpret_cast<unsigned int*>(ws + 2LL * planes + 2LL * planes * nblk);
    const float* base = x + (long long)p * hw;
    double s = 0, q = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (long long)nblk * blockDim.x) {
        const double v = base[i];
        s += v;
        q += v * v;
    }
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s; sh[1][threadIdx.x >> 5] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += sh[0][w]; b += sh[1][w]; }
        partial[((long long)p * nblk + blockIdx.x) * 2] = a;
        partial[((long long)p * nblk + blockIdx.x) * 2 + 1] = b;
        __threadfence();
        is_last = (atomicAdd(&tickets[2 * p], 1u) == (unsigned)(nblk - 1));
    }
    __syncthreads();
    if (is_last && threadIdx.x == 0) {
        __threadfence();
        double a = 0, b = 0;
        for (int k = 0; k < nblk; ++k) {
            a += __ldcg(&partial[((long long)p * nblk + k) * 2]);
            b += __ldcg(&partial[((long long)p * nblk + k) * 2 + 1]);
        }
        sums[2 * p] = a;
        sums[2 * p + 1] = b;
    }
}

// AdaIN (colorfix.py:45-71): out = (content - mean_c) / std_c * std_s + mean_s, std = sqrt(unbiased var + 1e-5)
__global__ void adain_apply_kernel(const float* __restrict__ content, const double* __restrict__ cs,
                                   const double* __restrict__ ss, float* __restrict__ out, long long hw, int planes) {
    const long long total = (long long)planes * hw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(i / hw);
        const double n = (double)hw;
        const double cm = cs[2 * p] / n, sm = ss[2 * p] / n;
        const double cv = (cs[2 * p + 1] - n * cm * cm) / (n - 1.0), sv = (ss[2 * p + 1] - n * sm * sm) / (n - 1.0);
        const float cstd = sqrtf((float)cv + 1e-5f), sstd = sqrtf((float)sv + 1e-5f);
        out[i] = (content[i] - (float)cm) / cstd * sstd + (float)sm;
    }
}

// Tensor2PIL (SUPIR/util.py:87-94): bicubic resize (torch interpolate, align_corners=False, A = -0.75, border indices clamped),
// then x * 127.5 + 127.5, clip to [0, 255], truncate to uint8, HWC. Same operation order as ATen's upsample_bicubic2d (rows
// first, then columns; coefficient polynomials as in aten/src/ATen/native/UpSample.h) so the bytes match torch's.
__device__ __forceinline__ float cubic_conv1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic_conv2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
__device__ __forceinline__ void cubic_coeffs(float t, float (&c)[4]) {
    const float A = -0.75f;
    c[0] = cubic_conv2(t + 1.0f, A);
    c[1] = cubic_conv1(t, A);
    const float u = 1.0f - t;
    c[2] = cubic_conv1(u, A);
    c[3] = cubic_conv2(u + 1.0f, A);
}
__global__ void image_to_uint8_bicubic_kernel(const float* __restrict__ x, int C, int H, int W, unsigned char* __restrict__ out,
                                              int h0, int w0, float scale_h, float scale_w) {
    const long long total = (long long)h0 * w0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % w0), oy = (int)(i / w0);
        const float rx = scale_w * (ox + 0.5f) - 0.5f, ry = scale_h * (oy + 0.5f) - 0.5f;
        const int ix = (int)floorf(rx), iy = (int)floorf(ry);
        float cx[4], cy[4];
        cubic_coeffs(rx - ix, cx);
        cubic_coeffs(ry - iy, cy);
        for (int c = 0; c < C; ++c) {
            const float* pl = x + (long long)c * H * W;
            float rows[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float* r = pl + (long long)min(max(iy - 1 + k, 0), H - 1) * W;
                rows[k] = r[min(max(ix - 1, 0), W - 1)] * cx[0] + r[min(max(ix, 0), W - 1)] * cx[1] +
                          r[min(max(ix + 1, 0), W - 1)] * cx[2] + r[min(max(ix + 2, 0), W - 1)] * cx[3];
            }
            float v = rows[0] * cy[0] + rows[1] * cy[1] + rows[2] * cy[2] + rows[3] * cy[3];
            v = v * 127.5f + 127.5f;
            v = fminf(fmaxf(v, 0.f), 255.f);
            out[i * C + c] = (unsigned char)v;           // truncation, like numpy's astype(np.uint8) on clipped values
        }
    }
}

static const int kStatBlocks = 64;

}  // namespace supir

using namespace supir;

extern "C" int supir_wavelet_level(const float* img, float* low, float* high, int planes, int H, int W, int radius,
                                   int accumulate, void* stream) {
    SUPIR_REQUIRE(img && low && img != low && planes > 0 && H > 0 && W > 0 && radius > 0, "supir_wavelet_level: bad args");
    const long long total = (long long)planes * H * W;
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)device_sm_count() * 16;
    if (blocks > cap) blocks = cap;
    wavelet_level_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(img, low, high, planes, H, W,
                                                                                              radius, accumulate);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" long long supir_plane_stats_workspace(int planes) { return 2LL * planes + 2LL * planes * kStatBlocks + planes; }

extern "C" int supir_plane_stats(const float* x, int planes, long long hw, double* ws, long long ws_doubles, void* stream) {
    SUPIR_REQUIRE(x && ws && planes > 0 && hw > 1, "supir_plane_stats: bad args");
    const long long need = supir_plane_stats_workspace(planes);
    SUPIR_REQUIRE(ws_doubles >= need, "supir_plane_stats: workspace of %lld doubles < %lld required", ws_doubles, need);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    SUPIR_CHECK_CUDA(cudaMemsetAsync(ws + need - planes, 0, sizeof(double) * planes, st));
    plane_stats_kernel<<<dim3(kStatBlocks, planes), 256, 0, st>>>(x, hw, ws, planes);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_adain_apply(const float* content, const double* content_stats, const double* style_stats, float* out,
                                 int planes, long long hw, void* stream) {
    SUPIR_REQUIRE(content && content_stats && style_stats && out, "supir_adain_apply: null pointer");
    const long long total = (long long)planes * hw;
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)device_sm_count() * 16;
    if (blocks > cap) blocks = cap;
    adain_apply_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(content, content_stats, style_stats,
                                                                                            out, hw, planes);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_image_to_uint8_bicubic(const float* x, int C, int H, int W, unsigned char* out, int h0, int w0, void* stream) {
    SUPIR_REQUIRE(x && out && C > 0 && H > 0 && W > 0 && h0 > 0 && w0 > 0, "supir_image_to_uint8_bicubic: bad args");
    const long long total = (long long)h0 * w0;
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16LL) blocks = device_sm_count() * 16LL;
    image_to_uint8_bicubic_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        x, C, H, W, out, h0, w0, (float)H / (float)h0, (float)W / (float)w0);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}
