// supir_b200 — convolutions whose channel count is too small for the tensor-core tile (K or N < 8):
// the network entry/exit layers. CUDA-core kernels, HBM-bound.
//   * conv3x3, Cin <= 8, fp32 strided NCHW in -> NHWC bf16 out : UNet/GLVControl conv_in and input_hint_block
//     (openaimodel.py:704; SUPIR_v0.py:325,482), VAE encoder conv_in 3->128 and decoder conv_in 4->512 (model.py:512-514,646-648)
//   * conv3x3, Cout <= 8, NHWC bf16 in -> fp32 strided NCHW out (optionally only a crop window, placed at an offset) :
//     UNet out 320->4 (openaimodel.py:947-953), VAE conv_out 512->8 / 128->3 (model.py:563-569,694-696) including the
//     tiled VAE's crop_valid_region + paste into the result canvas (tilevae.py:556-567, 946)
//   * conv1x1 on fp32 NCHW with Cin, Cout <= 8 : quant_conv / post_quant_conv (autoencoder.py:297-298)
// The 3x3 kernels are templated on the 16-bit storage type E (common.cuh): Bf16, or F16 for the _f16 entry points.
#include "common.cuh"
#include "supir_b200.h"

namespace supir {

// -------- Cin <= 8 : thread = (pixel, 8 output channels); weights in shared memory as [Cin*9][Cout] --------
template <class E>
__global__ void conv3x3_small_cin_kernel(const float* __restrict__ x, long long sb, long long sc, long long sy,
                                         const float* __restrict__ w, const float* __restrict__ bias,
                                         const typename E::T* __restrict__ res, long long ldr,
                                         typename E::T* __restrict__ out, long long ldo, int B, int H, int W, int Cin,
                                         int Cout) {
    extern __shared__ float ws[];  // [Cin*9][Cout]
    const int taps = Cin * 9;
    for (int i = threadIdx.x; i < taps * Cout; i += blockDim.x) {
        const int co = i / taps, t = i % taps;      // source layout [Cout][Cin][3][3]
        ws[t * Cout + co] = w[i];
    }
    __syncthreads();
    const int cgs = Cout >> 3;
    const long long total = (long long)B * H * W * cgs;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(i % cgs);
        const long long pix = i / cgs;
        const int xx = (int)(pix % W);
        const int yy = (int)((pix / W) % H);
        const int b = (int)(pix / ((long long)W * H));
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = bias ? bias[cg * 8 + j] : 0.f;
        for (int ci = 0; ci < Cin; ++ci) {
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const int y2 = yy + t / 3 - 1, x2 = xx + t % 3 - 1;
                if (y2 < 0 || y2 >= H || x2 < 0 || x2 >= W) continue;
                const float v = E::round(__ldg(x + b * sb + ci * sc + y2 * sy + x2));
                const float4 w0 = *reinterpret_cast<const float4*>(&ws[(ci * 9 + t) * Cout + cg * 8]);
                const float4 w1 = *reinterpret_cast<const float4*>(&ws[(ci * 9 + t) * Cout + cg * 8 + 4]);
                acc[0] += v * w0.x; acc[1] += v * w0.y; acc[2] += v * w0.z; acc[3] += v * w0.w;
                acc[4] += v * w1.x; acc[5] += v * w1.y; acc[6] += v * w1.z; acc[7] += v * w1.w;
            }
        }
        if (res) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(res + pix * ldr + cg * 8));
            const uint32_t wr[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 f = E::unpack2(wr[t]);
                acc[2 * t] = E::round(acc[2 * t]) + f.x;
                acc[2 * t + 1] = E::round(acc[2 * t + 1]) + f.y;
            }
        }
        uint4 o;
        o.x = E::pack2(acc[0], acc[1]); o.y = E::pack2(acc[2], acc[3]);
        o.z = E::pack2(acc[4], acc[5]); o.w = E::pack2(acc[6], acc[7]);
        *reinterpret_cast<uint4*>(out + pix * ldo + cg * 8) = o;
    }
}

// -------- Cin <= 8 as a tensor-core GEMM: im2col of the fp32 NCHW input into E rows [pixel][Cin*9 -> KP], zero padded ----
// (k = ci * 9 + tap, the flattening of the weight [Cout][Cin][3][3]); the GEMM kernel then does bias / residual / store.
template <class E>
__global__ void im2col_small_cin_kernel(const float* __restrict__ x, long long sb, long long sc, long long sy,
                                        typename E::T* __restrict__ out, long long ldo, int B, int H, int W, int Cin, int KP) {
    const int kv = KP >> 3;                       // 16-byte vectors per row
    const long long total = (long long)B * H * W * kv;
    const int taps = Cin * 9;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(i % kv);
        const long long pix = i / kv;
        const int xx = (int)(pix % W);
        const int r = (int)(pix / W);
        const int yy = r % H, b = r / H;
        float e[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = v * 8 + j;
            float val = 0.f;
            if (k < taps) {
                const int ci = k / 9, t = k - ci * 9;
                const int y2 = yy + t / 3 - 1, x2 = xx + t % 3 - 1;
                if (y2 >= 0 && y2 < H && x2 >= 0 && x2 < W) val = __ldg(x + b * sb + ci * sc + y2 * sy + x2);
            }
            e[j] = val;
        }
        uint4 o;
        o.x = E::pack2(e[0], e[1]); o.y = E::pack2(e[2], e[3]);
        o.z = E::pack2(e[4], e[5]); o.w = E::pack2(e[6], e[7]);
        *reinterpret_cast<uint4*>(out + pix * ldo + v * 8) = o;
    }
}

// -------- Cout <= 8 : one warp per output pixel; lanes split the (tap, channel-vector) products --------
template <int COUT, class E>
__global__ void conv3x3_small_cout_kernel(const typename E::T* __restrict__ x, long long ldx, const float* __restrict__ w,
                                          const float* __restrict__ bias, float* __restrict__ out, long long ob,
                                          long long oc, long long oy, int B, int H, int W, int Cin, int cy0, int cx0,
                                          int ch, int cw) {
    const int lane = threadIdx.x & 31;
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    const long long total = (long long)B * ch * cw;
    const int cv = Cin >> 3;
    for (long long pi = warp_id; pi < total; pi += nwarps) {
        const int xo = (int)(pi % cw);
        const int yo = (int)((pi / cw) % ch);
        const int b = (int)(pi / ((long long)cw * ch));
        const int yy = yo + cy0, xx = xo + cx0;
        float acc[COUT];
#pragma unroll
        for (int j = 0; j < COUT; ++j) acc[j] = 0.f;
        for (int t = 0; t < 9; ++t) {
            const int y2 = yy + t / 3 - 1, x2 = xx + t % 3 - 1;
            if (y2 < 0 || y2 >= H || x2 < 0 || x2 >= W) continue;  // warp-uniform
            const typename E::T* xp = x + (((long long)b * H + y2) * W + x2) * ldx;
            for (int v = lane; v < cv; v += 32) {
                const uint4 u = __ldg(reinterpret_cast<const uint4*>(xp + v * 8));
                const uint32_t wx[4] = {u.x, u.y, u.z, u.w};
                float xf[8];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 f = E::unpack2(wx[q]);
                    xf[2 * q] = f.x; xf[2 * q + 1] = f.y;
                }
#pragma unroll
                for (int j = 0; j < COUT; ++j) {
                    const float* wp = w + ((long long)j * 9 + t) * Cin + v * 8;   // layout [Cout][9][Cin]
                    const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
                    const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
                    acc[j] += xf[0] * w0.x + xf[1] * w0.y + xf[2] * w0.z + xf[3] * w0.w + xf[4] * w1.x + xf[5] * w1.y +
                              xf[6] * w1.z + xf[7] * w1.w;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < COUT; ++j) acc[j] = warp_sum(acc[j]);
        if (lane < COUT) {
            float v = 0.f;
#pragma unroll
            for (int j = 0; j < COUT; ++j)
                if (lane == j) v = acc[j];
            v = E::round(v + (bias ? bias[lane] : 0.f));
            out[b * ob + lane * oc + yo * oy + xo] = v;
        }
    }
}

// -------- 1x1, Cin/Cout <= 8 on fp32 NCHW --------
__global__ void conv1x1_small_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                     float* __restrict__ y, int B, int Cin, int Cout, long long HW, float in_scale) {
    const long long total = (long long)B * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i % HW;
        float xin[8];
        for (int c = 0; c < Cin; ++c) xin[c] = bf16_round(x[(b * Cin + c) * HW + p] * in_scale);
        for (int o = 0; o < Cout; ++o) {
            float a = bias ? bias[o] : 0.f;
            for (int c = 0; c < Cin; ++c) a += xin[c] * w[o * Cin + c];
            y[(b * Cout + o) * HW + p] = bf16_round(a);
        }
    }
}

}  // namespace supir

using namespace supir;

template <class E>
static int conv3x3_small_cin_impl(const char* who, const float* x, long long sb, long long sc, long long sy, const float* w,
                                  const float* bias, const void* residual, long long ldr, void* out, long long ldo, int B, int H,
                                  int W, int Cin, int Cout, void* stream) {
    SUPIR_REQUIRE(x && w && out, "%s: null pointer", who);
    SUPIR_REQUIRE(Cin >= 1 && Cin <= 8 && Cout % 8 == 0 && ldo % 8 == 0, "%s: Cin=%d Cout=%d unsupported", who, Cin, Cout);
    const size_t smem = (size_t)Cin * 9 * Cout * sizeof(float);
    SUPIR_REQUIRE(smem <= 160 * 1024, "%s: weights do not fit shared memory", who);
    static size_t max_set_dev[64] = {};
    size_t& max_set = max_set_dev[current_device_slot()];
    if (smem > 48 * 1024 && smem > max_set) {
        SUPIR_CHECK_CUDA(cudaFuncSetAttribute(conv3x3_small_cin_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        max_set = smem;
    }
    const long long total = (long long)B * H * W * (Cout >> 3);
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)device_sm_count() * 4;
    if (blocks > cap) blocks = cap;
    conv3x3_small_cin_kernel<E><<<(unsigned)blocks, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
        x, sb, sc, sy, w, bias, reinterpret_cast<const typename E::T*>(residual), ldr, reinterpret_cast<typename E::T*>(out),
        ldo, B, H, W, Cin, Cout);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_conv3x3_small_cin(const float* x, long long sb, long long sc, long long sy, const float* w,
                                       const float* bias, const void* residual, long long ldr, void* out, long long ldo,
                                       int B, int H, int W, int Cin, int Cout, void* stream) {
    return conv3x3_small_cin_impl<Bf16>("supir_conv3x3_small_cin", x, sb, sc, sy, w, bias, residual, ldr, out, ldo, B, H, W, Cin,
                                        Cout, stream);
}

extern "C" int supir_conv3x3_small_cin_f16(const float* x, long long sb, long long sc, long long sy, const float* w,
                                           const float* bias, const void* residual, long long ldr, void* out, long long ldo,
                                           int B, int H, int W, int Cin, int Cout, void* stream) {
    return conv3x3_small_cin_impl<F16>("supir_conv3x3_small_cin_f16", x, sb, sc, sy, w, bias, residual, ldr, out, ldo, B, H, W, Cin,
                                       Cout, stream);
}

template <class E>
static int im2col_small_cin_impl(const char* who, const float* x, long long sb, long long sc, long long sy, void* out, long long ldo,
                                 int B, int H, int W, int Cin, int KP, void* stream) {
    SUPIR_REQUIRE(x && out, "%s: null pointer", who);
    SUPIR_REQUIRE(Cin >= 1 && Cin <= 8 && KP % 8 == 0 && KP >= Cin * 9 && ldo >= KP && ldo % 8 == 0,
                  "%s: Cin=%d KP=%d unsupported", who, Cin, KP);
    const long long total = (long long)B * H * W * (KP >> 3);
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)device_sm_count() * 16;
    if (blocks > cap) blocks = cap;
    im2col_small_cin_kernel<E><<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        x, sb, sc, sy, reinterpret_cast<typename E::T*>(out), ldo, B, H, W, Cin, KP);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_im2col_3x3_small_cin(const float* x, long long sb, long long sc, long long sy, void* out, long long ldo,
                                          int B, int H, int W, int Cin, int KP, void* stream) {
    return im2col_small_cin_impl<Bf16>("supir_im2col_3x3_small_cin", x, sb, sc, sy, out, ldo, B, H, W, Cin, KP, stream);
}

extern "C" int supir_im2col_3x3_small_cin_f16(const float* x, long long sb, long long sc, long long sy, void* out, long long ldo,
                                              int B, int H, int W, int Cin, int KP, void* stream) {
    return im2col_small_cin_impl<F16>("supir_im2col_3x3_small_cin_f16", x, sb, sc, sy, out, ldo, B, H, W, Cin, KP, stream);
}

template <class E>
static int conv3x3_small_cout_impl(const char* who, const void* x, long long ldx, const float* w, const float* bias, float* out,
                                   long long ob, long long oc, long long oy, int B, int H, int W, int Cin, int Cout,
                                   int crop_y0, int crop_x0, int crop_h, int crop_w, void* stream) {
    SUPIR_REQUIRE(x && w && out, "%s: null pointer", who);
    SUPIR_REQUIRE(Cin % 8 == 0 && ldx % 8 == 0, "%s: Cin must be a multiple of 8", who);
    SUPIR_REQUIRE(crop_y0 >= 0 && crop_x0 >= 0 && crop_y0 + crop_h <= H && crop_x0 + crop_w <= W && crop_h > 0 && crop_w > 0,
                  "%s: crop window outside the tile", who);
    const long long total = (long long)B * crop_h * crop_w;
    long long blocks = (total + 7) / 8;
    const long long cap = (long long)device_sm_count() * 16;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const typename E::T* xp = reinterpret_cast<const typename E::T*>(x);
#define LAUNCH(CO)                                                                                                       \
    conv3x3_small_cout_kernel<CO, E><<<(unsigned)blocks, 256, 0, st>>>(xp, ldx, w, bias, out, ob, oc, oy, B, H, W, Cin, \
                                                                       crop_y0, crop_x0, crop_h, crop_w)
    if (Cout == 3) LAUNCH(3);
    else if (Cout == 4) LAUNCH(4);
    else if (Cout == 8) LAUNCH(8);
    else return set_error(SUPIR_ERR_UNSUPPORTED, "%s: Cout=%d unsupported (3, 4, 8)", who, Cout);
#undef LAUNCH
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_conv3x3_small_cout(const void* x, long long ldx, const float* w, const float* bias, float* out,
                                        long long ob, long long oc, long long oy, int B, int H, int W, int Cin, int Cout,
                                        int crop_y0, int crop_x0, int crop_h, int crop_w, void* stream) {
    return conv3x3_small_cout_impl<Bf16>("supir_conv3x3_small_cout", x, ldx, w, bias, out, ob, oc, oy, B, H, W, Cin, Cout, crop_y0,
                                         crop_x0, crop_h, crop_w, stream);
}

extern "C" int supir_conv3x3_small_cout_f16(const void* x, long long ldx, const float* w, const float* bias, float* out,
                                            long long ob, long long oc, long long oy, int B, int H, int W, int Cin, int Cout,
                                            int crop_y0, int crop_x0, int crop_h, int crop_w, void* stream) {
    return conv3x3_small_cout_impl<F16>("supir_conv3x3_small_cout_f16", x, ldx, w, bias, out, ob, oc, oy, B, H, W, Cin, Cout,
                                        crop_y0, crop_x0, crop_h, crop_w, stream);
}

extern "C" int supir_conv1x1_small_nchw(const float* x, const float* w, const float* bias, float* y, int B, int Cin,
                                        int Cout, long long HW, float in_scale, void* stream) {
    SUPIR_REQUIRE(x && w && y && Cin >= 1 && Cin <= 8 && Cout >= 1 && Cout <= 8, "supir_conv1x1_small_nchw: bad args");
    const long long total = (long long)B * HW;
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)device_sm_count() * 8;
    if (blocks > cap) blocks = cap;
    conv1x1_small_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, w, bias, y, B, Cin, Cout, HW, in_scale);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}
