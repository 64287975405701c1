// supir_b200 — K1/K5/K13 of SURVEY.md §2a: GroupNorm(32) [+SiLU], LayerNorm, tiled-VAE cross-tile GroupNorm.
// All HBM-bound: 128-bit loads/stores on channels-last 16-bit data, fp32 math, fp64 cross-block sums. The diffusion-network
// kernels are templated on the storage type E (common.cuh): Bf16, or F16 for the _f16 entry points.
//
// Reference call sites: GroupNorm32 (sgm/modules/diffusionmodules/util.py:258-276, eps 1e-5) in ResBlock
// (openaimodel.py:260-264,295-308), ZeroSFT/ZeroCrossAttn (SUPIR/modules/SUPIR_v0.py:72,110,128-129);
// attention.Normalize / VAE Normalize (attention.py:122-125, model.py:49-52, eps 1e-6); nn.LayerNorm
// (attention.py:437-439); tiled VAE statistics merge (SUPIR/utils/tilevae.py:511-553, 599-648).
#include "common.cuh"
#include "supir_b200.h"

namespace supir {

// ---------------------------------------------------------------------------------------------
// GroupNorm statistics: per (image, group) sum and sum of squares in fp64 — deterministic (no floating-point atomics):
// block = KP pixels x (C/8) channel-vectors; per-thread fp32 partials over a pixel chunk -> fixed-order shared-memory
// reduction -> per-block fp64 group partials in the workspace; the last block of an image to finish (integer ticket)
// adds the block partials in block order into sums[b, g, 0:2].
// workspace layout (doubles): [B*G*2 final sums][B*nblk*G*2 block partials][B tickets (as uint32 in 8-byte slots)]
// ---------------------------------------------------------------------------------------------
template <class E>
__global__ void gn_stats_kernel(const typename E::T* __restrict__ x, long long ldx, int HW, int C, int G,
                                int pixels_per_block, double* __restrict__ ws, int B) {
    extern __shared__ float sm[];  // [2][kp][C]
    __shared__ int is_last;
    const int cv_count = C >> 3;
    const int kp = blockDim.x / cv_count;
    const int cv = threadIdx.x % cv_count;
    const int pl = threadIdx.x / cv_count;
    const int b = blockIdx.y;
    const int nblk = gridDim.x;
    const int p0 = blockIdx.x * pixels_per_block;
    const int p1 = min(p0 + pixels_per_block, HW);
    double* sums = ws;
    double* partial = ws + (long long)B * G * 2;
    unsigned int* tickets = reinterpret_cast<unsigned int*>(ws + (long long)B * G * 2 + (long long)B * nblk * G * 2);
    float s[8], ss[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = ss[j] = 0.f;
    const typename E::T* base = x + ((long long)b * HW) * ldx + cv * 8;
    for (int p = p0 + pl; p < p1; p += kp) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(base + (long long)p * ldx));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = E::unpack2(w[t]);
            s[2 * t] += f.x; ss[2 * t] += f.x * f.x;
            s[2 * t + 1] += f.y; ss[2 * t + 1] += f.y * f.y;
        }
    }
    float* sm_s = sm;
    float* sm_q = sm + kp * C;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sm_s[pl * C + cv * 8 + j] = s[j];
        sm_q[pl * C + cv * 8 + j] = ss[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float a = 0.f, q = 0.f;
        for (int r = 0; r < kp; ++r) { a += sm_s[r * C + c]; q += sm_q[r * C + c]; }
        sm_s[c] = a;   // row 0, own column only
        sm_q[c] = q;
    }
    __syncthreads();
    const int cpg = C / G;
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        double a = 0, q = 0;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) { a += sm_s[c]; q += sm_q[c]; }
        double* dst = partial + (((long long)b * nblk + blockIdx.x) * G + g) * 2;
        dst[0] = a;
        dst[1] = q;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(&tickets[2 * b], 1u) == (unsigned)(nblk - 1));
    __syncthreads();
    if (is_last) {
        __threadfence();
        // block partials -> final sums, in a fixed order: `lanes` threads per group each add every lanes-th partial in block
        // order, then the lanes' subtotals are added in lane order (deterministic, and not a serial walk over all blocks)
        double* red = reinterpret_cast<double*>(sm);            // [blockDim.x][2], fits: 2*kp*C floats >= 4*blockDim.x
        int lanes = blockDim.x / G;
        if (lanes < 1) lanes = 1;
        const int gpp = blockDim.x / lanes;                     // groups handled per pass
        const int l = threadIdx.x % lanes;
        for (int g0 = 0; g0 < G; g0 += gpp) {
            const int g = g0 + threadIdx.x / lanes;
            double a = 0, q = 0;
            if (g < G && threadIdx.x < gpp * lanes) {
                for (int k = l; k < nblk; k += lanes) {
                    const double* src = partial + (((long long)b * nblk + k) * G + g) * 2;
                    a += __ldcg(src);
                    q += __ldcg(src + 1);
                }
            }
            __syncthreads();
            red[2 * threadIdx.x] = a;
            red[2 * threadIdx.x + 1] = q;
            __syncthreads();
            if (g < G && l == 0 && threadIdx.x < gpp * lanes) {
                double ta = 0, tq = 0;
                for (int i = 0; i < lanes; ++i) { ta += red[2 * (threadIdx.x + i)]; tq += red[2 * (threadIdx.x + i) + 1]; }
                sums[((long long)b * G + g) * 2] = ta;
                sums[((long long)b * G + g) * 2 + 1] = tq;
            }
        }
    }
}

// sums -> (mean, biased var) per (image, group)
__global__ void gn_finalize_kernel(const double* __restrict__ sums, int n, double count, float* __restrict__ mean,
                                   float* __restrict__ var) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double m = sums[2 * i] / count;
    double v = sums[2 * i + 1] / count - m * m;
    if (v < 0) v = 0;
    mean[i] = (float)m;
    var[i] = (float)v;
}

// tiled VAE: pixel-count-weighted average of per-tile mean AND var (the reference's approximation, tilevae.py:629-648)
__global__ void gn_merge_tiles_kernel(const float* __restrict__ tile_mean, const float* __restrict__ tile_var,
                                      const float* __restrict__ weights, int T, int n, float* __restrict__ mean,
                                      float* __restrict__ var) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float m = 0.f, v = 0.f;
    for (int t = 0; t < T; ++t) {  // same summation order as torch.sum over the tile dimension
        m += tile_mean[(long long)t * n + i] * weights[t];
        v += tile_var[(long long)t * n + i] * weights[t];
    }
    mean[i] = m;
    var[i] = v;
}

// Per-thread scale / shift of one 8-channel vector: y = x * sc + sh with sc = rstd * gamma, sh = beta - mean * sc.
// Statistics come either as fp64 (sum, sumsq) pairs or as fp32 (mean, biased var).
__device__ __forceinline__ void gn_scale_shift(int b, int c0, int C, int G, const double* __restrict__ sums, double count,
                                               const float* __restrict__ mean, const float* __restrict__ var,
                                               const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                               float (&sc)[8], float (&sh)[8]) {
    const int cpg = C / G;
    int g_prev = -1;
    float m = 0.f, rstd = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        const int g = c / cpg;
        if (g != g_prev) {
            float v;
            if (sums) {
                const double dm = sums[((long long)b * G + g) * 2] / count;
                double dv = sums[((long long)b * G + g) * 2 + 1] / count - dm * dm;
                if (dv < 0) dv = 0;
                m = (float)dm; v = (float)dv;
            } else {
                m = mean[b * G + g]; v = var[b * G + g];
            }
            rstd = rsqrtf(v + eps);
            g_prev = g;
        }
        sc[j] = rstd * (gamma ? gamma[c] : 1.f);
        sh[j] = (beta ? beta[c] : 0.f) - m * sc[j];
    }
}

// y = (x - mean) * rsqrt(var + eps) * gamma + beta [-> SiLU] ; E in, E out, channels-last.
// block = kp pixel lanes x (C/8) channel vectors; a thread keeps its vector's scale / shift in registers and walks pixels.
template <class E>
__global__ void gn_apply_kernel(const typename E::T* __restrict__ x, long long ldx, typename E::T* __restrict__ y,
                                long long ldy, int HW, int C, int G, const float* __restrict__ mean,
                                const float* __restrict__ var, const double* __restrict__ sums, double count,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int silu,
                                int pixels_per_block) {
    const int cv_count = C >> 3;
    const int kp = blockDim.x / cv_count;
    const int cv = threadIdx.x % cv_count;
    const int pl = threadIdx.x / cv_count;
    const int b = blockIdx.y;
    float sc[8], sh[8];
    gn_scale_shift(b, cv * 8, C, G, sums, count, mean, var, gamma, beta, eps, sc, sh);
    const int p0 = blockIdx.x * pixels_per_block;
    const int p1 = min(p0 + pixels_per_block, HW);
    const typename E::T* xb = x + ((long long)b * HW) * ldx + cv * 8;
    typename E::T* yb = y + ((long long)b * HW) * ldy + cv * 8;
    auto one = [&](const uint4 u, long long p) {
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
        uint32_t o[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = E::unpack2(w[t]);
            float a = f.x * sc[2 * t] + sh[2 * t];
            float d = f.y * sc[2 * t + 1] + sh[2 * t + 1];
            if (silu) { a = silu_f(a); d = silu_f(d); }
            o[t] = E::pack2(a, d);
        }
        __stcs(reinterpret_cast<uint4*>(yb + p * ldy), make_uint4(o[0], o[1], o[2], o[3]));
    };
    int p = p0 + pl;
    for (; p + 3 * kp < p1; p += 4 * kp) {      // four independent 16-byte loads in flight per thread
        const uint4 u0 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)p * ldx));
        const uint4 u1 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)(p + kp) * ldx));
        const uint4 u2 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)(p + 2 * kp) * ldx));
        const uint4 u3 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)(p + 3 * kp) * ldx));
        one(u0, p); one(u1, p + kp); one(u2, p + 2 * kp); one(u3, p + 3 * kp);
    }
    for (; p < p1; p += kp) one(__ldg(reinterpret_cast<const uint4*>(xb + (long long)p * ldx)), p);
}

// ---------------------------------------------------------------------------------------------
// GroupNorm [+ SiLU] apply written as e4m3 for supir_conv3x3_fp8 (the ResBlocks' 3x3 convolutions in the FP8 convs mode): codes
// q [B*HW, ldq] and one scale per image, scale[b] = amax / 448 over that image's fp32 apply values (e4m3_row_scale; no 16-bit
// rounding in between). Two passes over x: gn_amax_kernel folds each block's max |value| into amax[b] (atomicMax on the bits
// of a non-negative float: a max does not depend on the order, so the result is deterministic), then gn_apply_quant_kernel
// computes the same fp32 values again (gn_value, the arithmetic of gn_apply_kernel) and writes the codes. Per-image scales
// keep the images of a batch independent of each other. Same block layout as gn_apply_kernel.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float gn_value(float v, float sc, float sh, int silu) {
    const float a = v * sc + sh;
    return silu ? silu_f(a) : a;
}

__global__ void gn_amax_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int HW, int C, int G,
                               const double* __restrict__ sums, double count, const float* __restrict__ gamma,
                               const float* __restrict__ beta, float eps, int silu, int pixels_per_block,
                               unsigned int* __restrict__ amax) {
    __shared__ unsigned int block_max;
    const int cv_count = C >> 3;
    const int kp = blockDim.x / cv_count;
    const int cv = threadIdx.x % cv_count;
    const int pl = threadIdx.x / cv_count;            // >= kp: a thread of the last warp's padding, no pixels
    const int b = blockIdx.y;
    if (threadIdx.x == 0) block_max = 0u;
    float sc[8], sh[8];
    gn_scale_shift(b, cv * 8, C, G, sums, count, nullptr, nullptr, gamma, beta, eps, sc, sh);
    const int p0 = blockIdx.x * pixels_per_block;
    const int p1 = min(p0 + pixels_per_block, HW);
    const __nv_bfloat16* xb = x + ((long long)b * HW) * ldx + cv * 8;
    float m = 0.f;
    for (int p = p0 + pl; pl < kp && p < p1; p += kp) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(xb + (long long)p * ldx));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = unpack_bf16x2(w[t]);
            m = fmaxf(m, fmaxf(fabsf(gn_value(f.x, sc[2 * t], sh[2 * t], silu)), fabsf(gn_value(f.y, sc[2 * t + 1], sh[2 * t + 1], silu))));
        }
    }
    m = warp_max(m);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) atomicMax(&block_max, __float_as_uint(m));
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(amax + b, block_max);
}

__global__ void gn_apply_quant_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, uint8_t* __restrict__ q, long long ldq,
                                      float* __restrict__ scale, const unsigned int* __restrict__ amax, int HW, int C, int G,
                                      const double* __restrict__ sums, double count, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, float eps, int silu, int pixels_per_block) {
    const int cv_count = C >> 3;
    const int kp = blockDim.x / cv_count;
    const int cv = threadIdx.x % cv_count;
    const int pl = threadIdx.x / cv_count;
    const int b = blockIdx.y;
    float s, inv;
    e4m3_row_scale(__uint_as_float(amax[b]), s, inv);
    if (blockIdx.x == 0 && threadIdx.x == 0) scale[b] = s;
    float sc[8], sh[8];
    gn_scale_shift(b, cv * 8, C, G, sums, count, nullptr, nullptr, gamma, beta, eps, sc, sh);
    const int p0 = blockIdx.x * pixels_per_block;
    const int p1 = min(p0 + pixels_per_block, HW);
    const __nv_bfloat16* xb = x + ((long long)b * HW) * ldx + cv * 8;
    uint8_t* qb = q + ((long long)b * HW) * ldq + cv * 8;
    auto one = [&](const uint4 u, long long p) {
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
        float v[8];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = unpack_bf16x2(w[t]);
            v[2 * t] = gn_value(f.x, sc[2 * t], sh[2 * t], silu) * inv;
            v[2 * t + 1] = gn_value(f.y, sc[2 * t + 1], sh[2 * t + 1], silu) * inv;
        }
        __stcs(reinterpret_cast<uint2*>(qb + p * ldq), make_uint2(pack_e4m3x4(v[0], v[1], v[2], v[3]), pack_e4m3x4(v[4], v[5], v[6], v[7])));
    };
    int p = p0 + pl;
    for (; p + 3 * kp < p1; p += 4 * kp) {      // four independent 16-byte loads in flight per thread
        const uint4 u0 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)p * ldx));
        const uint4 u1 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)(p + kp) * ldx));
        const uint4 u2 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)(p + 2 * kp) * ldx));
        const uint4 u3 = __ldg(reinterpret_cast<const uint4*>(xb + (long long)(p + 3 * kp) * ldx));
        one(u0, p); one(u1, p + kp); one(u2, p + 2 * kp); one(u3, p + 3 * kp);
    }
    for (; p < p1; p += kp) one(__ldg(reinterpret_cast<const uint4*>(xb + (long long)p * ldx)), p);
}

// ---------------------------------------------------------------------------------------------
// ZeroSFT tail (SUPIR_v0.py:110-113): out = lerp(h_raw, GN(h) * (gamma + 1) + beta, control_scale)
//   h      : [B, HW, C]  (= cat(h_ori, skip + zero_conv(c)))        gb : [B, HW, 2C] = (gamma | beta) conv outputs
//   h_raw first C1 channels equal h's; the remaining C - C1 come from `skip_raw` [B, HW, C - C1]
// ---------------------------------------------------------------------------------------------
template <class E>
__global__ void sft_apply_kernel(const typename E::T* __restrict__ h, long long ldh,
                                 const typename E::T* __restrict__ skip_raw, long long lds, int C1,
                                 const typename E::T* __restrict__ gb, long long ldgb, typename E::T* __restrict__ out,
                                 long long ldo, int HW, int C, int G, const double* __restrict__ sums, double count,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 const float* __restrict__ control_scale, int pixels_per_block) {
    const int cv_count = C >> 3;
    const int kp = blockDim.x / cv_count;
    const int cv = threadIdx.x % cv_count;
    const int pl = threadIdx.x / cv_count;
    const int b = blockIdx.y;
    const int c0 = cv * 8;
    float sc[8], sh[8];
    gn_scale_shift(b, c0, C, G, sums, count, nullptr, nullptr, gamma, beta, eps, sc, sh);
    const float cs = *control_scale;
    const int p0 = blockIdx.x * pixels_per_block;
    const int p1 = min(p0 + pixels_per_block, HW);
    const bool from_skip = c0 >= C1;
    auto one = [&](int p) {
        const long long row = (long long)b * HW + p;
        const uint4 uh = __ldg(reinterpret_cast<const uint4*>(h + row * ldh + c0));
        const uint4 ug = __ldg(reinterpret_cast<const uint4*>(gb + row * ldgb + c0));
        const uint4 ub = __ldg(reinterpret_cast<const uint4*>(gb + row * ldgb + C + c0));
        uint4 ur = uh;
        if (from_skip) ur = __ldg(reinterpret_cast<const uint4*>(skip_raw + row * lds + (c0 - C1)));
        const uint32_t wh[4] = {uh.x, uh.y, uh.z, uh.w}, wg[4] = {ug.x, ug.y, ug.z, ug.w},
                       wb[4] = {ub.x, ub.y, ub.z, ub.w}, wr[4] = {ur.x, ur.y, ur.z, ur.w};
        uint32_t o[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 fh = E::unpack2(wh[t]), fg = E::unpack2(wg[t]), fb = E::unpack2(wb[t]), fr = E::unpack2(wr[t]);
            // normalised (fp32) * (gamma + 1) + beta, each intermediate rounded like the reference's 16-bit tensors
            const float n0 = fh.x * sc[2 * t] + sh[2 * t], n1 = fh.y * sc[2 * t + 1] + sh[2 * t + 1];
            const float a = n0 * (E::round(fg.x + 1.f)) + fb.x;
            const float d = n1 * (E::round(fg.y + 1.f)) + fb.y;
            o[t] = E::pack2(a * cs + fr.x * (1.f - cs), d * cs + fr.y * (1.f - cs));
        }
        __stcs(reinterpret_cast<uint4*>(out + row * ldo + c0), make_uint4(o[0], o[1], o[2], o[3]));
    };
    int p = p0 + pl;
    for (; p + kp < p1; p += 2 * kp) { one(p); one(p + kp); }
    for (; p < p1; p += kp) one(p);
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over the last dim (C <= 2048, C % 8 == 0): one warp per row, row kept in registers.
// QUANT: the normalised row is written as e4m3 codes qout [rows, ldq] plus a row scale qscale[row] (e4m3_row_scale of the fp32
// values' amax), for supir_gemm_fp8: no intermediate 16-bit rounding, and y is not written.
// ---------------------------------------------------------------------------------------------
template <int MAXV, class E, bool QUANT = false>  // max 16-byte vectors per lane
__global__ void layernorm_kernel(const typename E::T* __restrict__ x, long long ldx, typename E::T* __restrict__ y,
                                 long long ldy, long long rows, int C, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float eps, float2* __restrict__ stats,
                                 uint8_t* __restrict__ qout = nullptr, long long ldq = 0, float* __restrict__ qscale = nullptr) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int nv = C >> 3;
    // a warp walks rows with stride nwarps; the next row's loads are issued before this row's reductions, so the two warp
    // reductions between load and store no longer leave the memory pipe idle
    uint4 nxt[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < nv) nxt[i] = __ldg(reinterpret_cast<const uint4*>(x + row * ldx + vi * 8));
    }
    for (; row < rows; row += nwarps) {
        float v[MAXV][8];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < nv) {
                const uint32_t w[4] = {nxt[i].x, nxt[i].y, nxt[i].z, nxt[i].w};
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const float2 f = E::unpack2(w[t]);
                    v[i][2 * t] = f.x; v[i][2 * t + 1] = f.y;
                    s += f.x + f.y;
                }
            }
        }
        const long long nrow = row + nwarps;
        if (nrow < rows) {
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                const int vi = lane + i * 32;
                if (vi < nv) nxt[i] = __ldg(reinterpret_cast<const uint4*>(x + nrow * ldx + vi * 8));
            }
        }
        const float mean = warp_sum(s) / C;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < nv) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q += d * d; }
            }
        }
        const float rstd = rsqrtf(warp_sum(q) / C + eps);
        if (stats) {                                   // statistics only (LayerNorm folded into the consumer GEMM's epilogue)
            if (lane == 0) stats[row] = make_float2(rstd, mean * rstd);
            continue;
        }
        if constexpr (QUANT) {
            float amax = 0.f;
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                const int vi = lane + i * 32;
                if (vi < nv) {
                    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8));
                    const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8 + 4));
                    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8));
                    const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8 + 4));
                    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        v[i][j] = (v[i][j] - mean) * rstd * gg[j] + bb[j];
                        amax = fmaxf(amax, fabsf(v[i][j]));
                    }
                }
            }
            float sc, inv;
            e4m3_row_scale(warp_max(amax), sc, inv);
            if (lane == 0) qscale[row] = sc;
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                const int vi = lane + i * 32;
                if (vi < nv) {
                    const uint32_t lo = pack_e4m3x4(v[i][0] * inv, v[i][1] * inv, v[i][2] * inv, v[i][3] * inv);
                    const uint32_t hi = pack_e4m3x4(v[i][4] * inv, v[i][5] * inv, v[i][6] * inv, v[i][7] * inv);
                    __stcs(reinterpret_cast<uint2*>(qout + row * ldq + vi * 8), make_uint2(lo, hi));
                }
            }
            continue;
        }
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < nv) {
                const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8));
                const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8 + 4));
                const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8));
                const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8 + 4));
                const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
                uint32_t o[4];
#pragma unroll
                for (int t = 0; t < 4; ++t)
                    o[t] = E::pack2((v[i][2 * t] - mean) * rstd * gg[2 * t] + bb[2 * t],
                                    (v[i][2 * t + 1] - mean) * rstd * gg[2 * t + 1] + bb[2 * t + 1]);
                __stcs(reinterpret_cast<uint4*>(y + row * ldy + vi * 8), make_uint4(o[0], o[1], o[2], o[3]));
            }
        }
    }
}

// row softmax for the materialised single-head VAE attention: P = softmax(S * scale), fp32 in, bf16 out.
// One block per row; the row is read from HBM once (128-bit loads) into shared memory, exponentiated in place, and written
// once as bf16 (the generic kernel below re-reads the row from global memory and serves rows that do not fit or align).
__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : (is_max ? -INFINITY : 0.f);
        t = is_max ? warp_max(t) : warp_sum(t);
        if (threadIdx.x == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}

__global__ void softmax_rows_smem_kernel(const float* __restrict__ S, long long lds, __nv_bfloat16* __restrict__ P,
                                         long long ldp, int cols, float scale) {
    extern __shared__ float rowbuf[];      // cols rounded up to 8
    __shared__ float red[33];
    const long long row = blockIdx.x;
    const float4* s4 = reinterpret_cast<const float4*>(S + row * lds);
    const int n4 = cols >> 2;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = __ldcs(s4 + i);
        reinterpret_cast<float4*>(rowbuf)[i] = v;
        m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
    }
    for (int c = (n4 << 2) + threadIdx.x; c < cols; c += blockDim.x) {
        const float v = S[row * lds + c];
        rowbuf[c] = v;
        m = fmaxf(m, v);
    }
    m = block_reduce(m, red, true);
    float sum = 0.f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) {
        const float e = __expf((rowbuf[c] - m) * scale);
        rowbuf[c] = e;
        sum += e;
    }
    sum = block_reduce(sum, red, false);
    const float inv = 1.f / sum;
    __nv_bfloat16* p = P + row * ldp;
    const int n8 = cols >> 3;
    for (int i = threadIdx.x; i < n8; i += blockDim.x) {
        const float4 a = reinterpret_cast<const float4*>(rowbuf)[2 * i], c = reinterpret_cast<const float4*>(rowbuf)[2 * i + 1];
        uint4 u;
        u.x = pack_bf16x2(a.x * inv, a.y * inv);
        u.y = pack_bf16x2(a.z * inv, a.w * inv);
        u.z = pack_bf16x2(c.x * inv, c.y * inv);
        u.w = pack_bf16x2(c.z * inv, c.w * inv);
        reinterpret_cast<uint4*>(p)[i] = u;
    }
    for (int c = (n8 << 3) + threadIdx.x; c < cols; c += blockDim.x) p[c] = __float2bfloat16_rn(rowbuf[c] * inv);
}

__global__ void softmax_rows_kernel(const float* __restrict__ S, long long lds, __nv_bfloat16* __restrict__ P,
                                    long long ldp, int cols, float scale) {
    const long long row = blockIdx.x;
    const float* s = S + row * lds;
    __shared__ float red[33];
    float m = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, s[c]);
    m = block_reduce(m, red, true);
    float sum = 0.f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) sum += __expf((s[c] - m) * scale);
    sum = block_reduce(sum, red, false);
    const float inv = 1.f / sum;
    __nv_bfloat16* p = P + row * ldp;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) p[c] = __float2bfloat16_rn(__expf((s[c] - m) * scale) * inv);
}

static int gn_launch_shape(int HW, int C, int& threads, int& ppb, int& blocks_x) {
    const int cv = C >> 3;
    int kp = 512 / cv;
    if (kp < 1) kp = 1;
    threads = kp * cv;
    // enough blocks to cover the machine a few times, but at least 32 pixels per thread-row to amortise the reduction
    ppb = kp * 16;
    if (ppb < 64) ppb = 64;
    // very large images (tiled VAE): at most ~592 blocks per image (4 per SM). Depends on (HW, C) only, never on the batch:
    // a window-sharded run must add in the same order as the unsharded one.
    const int cap = (HW + 591) / 592;
    if (ppb < cap) ppb = (cap + kp - 1) / kp * kp;
    blocks_x = (HW + ppb - 1) / ppb;
    return 0;
}

}  // namespace supir

using namespace supir;

extern "C" long long supir_groupnorm_stats_workspace(int B, int HW, int C, int groups) {
    if (C % 8 != 0 || C <= 0) return -1;
    int threads, ppb, bx;
    gn_launch_shape(HW, C, threads, ppb, bx);
    return (long long)B * groups * 2 + (long long)B * bx * groups * 2 + B;
}

template <class E>
static int groupnorm_stats_impl(const char* who, const void* x, long long ldx, int B, int HW, int C, int groups, double* ws,
                                long long ws_doubles, void* stream) {
    SUPIR_REQUIRE(x && ws, "%s: null pointer", who);
    SUPIR_REQUIRE(C % 8 == 0 && C % groups == 0 && ldx % 8 == 0 && C <= 8192, "%s: bad C=%d", who, C);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int threads, ppb, bx;
    gn_launch_shape(HW, C, threads, ppb, bx);
    const long long need = (long long)B * groups * 2 + (long long)B * bx * groups * 2 + B;
    SUPIR_REQUIRE(ws_doubles >= need, "%s: workspace of %lld doubles < %lld required", who, ws_doubles, need);
    SUPIR_CHECK_CUDA(cudaMemsetAsync(ws + need - B, 0, sizeof(double) * B, st));   // tickets
    const int kp = threads / (C >> 3);
    const size_t smem = (size_t)2 * kp * C * sizeof(float);
    static size_t max_set_dev[64] = {};
    size_t& max_set = max_set_dev[current_device_slot()];
    if (smem > 48 * 1024 && smem > max_set) {
        SUPIR_CHECK_CUDA(cudaFuncSetAttribute(gn_stats_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        max_set = smem;
    }
    gn_stats_kernel<E><<<dim3(bx, B), threads, smem, st>>>(reinterpret_cast<const typename E::T*>(x), ldx, HW, C, groups, ppb, ws, B);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_groupnorm_stats(const void* x, long long ldx, int B, int HW, int C, int groups, double* ws,
                                     long long ws_doubles, void* stream) {
    return groupnorm_stats_impl<Bf16>("supir_groupnorm_stats", x, ldx, B, HW, C, groups, ws, ws_doubles, stream);
}

extern "C" int supir_groupnorm_stats_f16(const void* x, long long ldx, int B, int HW, int C, int groups, double* ws,
                                         long long ws_doubles, void* stream) {
    return groupnorm_stats_impl<F16>("supir_groupnorm_stats_f16", x, ldx, B, HW, C, groups, ws, ws_doubles, stream);
}

extern "C" int supir_groupnorm_finalize(const double* sums, int n, double count, float* mean, float* var, void* stream) {
    SUPIR_REQUIRE(sums && mean && var && n > 0, "supir_groupnorm_finalize: bad args");
    gn_finalize_kernel<<<(n + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(sums, n, count, mean, var);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_groupnorm_merge_tiles(const float* tile_mean, const float* tile_var, const float* weights, int T,
                                           int n, float* mean, float* var, void* stream) {
    SUPIR_REQUIRE(tile_mean && tile_var && weights && mean && var && T > 0 && n > 0, "supir_groupnorm_merge_tiles: bad args");
    gn_merge_tiles_kernel<<<(n + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(tile_mean, tile_var,
                                                                                              weights, T, n, mean, var);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

template <class E>
static int groupnorm_apply_impl(const char* who, const void* x, long long ldx, void* y, long long ldy, int B, int HW, int C,
                                int groups, const double* sums, const float* mean, const float* var, const float* gamma,
                                const float* beta, float eps, int silu, void* stream) {
    SUPIR_REQUIRE(x && y && (sums || (mean && var)), "%s: null pointer", who);
    SUPIR_REQUIRE(C % 8 == 0 && C % groups == 0 && ldx % 8 == 0 && ldy % 8 == 0 && C <= 8192, "%s: bad C=%d", who, C);
    const int cvc = C >> 3;
    int kp = 512 / cvc;
    if (kp < 1) kp = 1;
    const int threads = kp * cvc;
    int ppb = kp * 32;              // 32 pixels per thread amortise the per-thread scale / shift set-up
    if (ppb > HW) ppb = (HW + kp - 1) / kp * kp;
    const int bx = (HW + ppb - 1) / ppb;
    gn_apply_kernel<E><<<dim3(bx, B), threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const typename E::T*>(x), ldx, reinterpret_cast<typename E::T*>(y), ldy, HW, C, groups, mean,
        var, sums, (double)HW * (C / groups), gamma, beta, eps, silu, ppb);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_groupnorm_apply(const void* x, long long ldx, void* y, long long ldy, int B, int HW, int C,
                                     int groups, const double* sums, const float* mean, const float* var,
                                     const float* gamma, const float* beta, float eps, int silu, void* stream) {
    return groupnorm_apply_impl<Bf16>("supir_groupnorm_apply", x, ldx, y, ldy, B, HW, C, groups, sums, mean, var, gamma, beta,
                                      eps, silu, stream);
}

extern "C" int supir_groupnorm_apply_f16(const void* x, long long ldx, void* y, long long ldy, int B, int HW, int C,
                                         int groups, const double* sums, const float* mean, const float* var,
                                         const float* gamma, const float* beta, float eps, int silu, void* stream) {
    return groupnorm_apply_impl<F16>("supir_groupnorm_apply_f16", x, ldx, y, ldy, B, HW, C, groups, sums, mean, var, gamma, beta,
                                     eps, silu, stream);
}

extern "C" int supir_groupnorm_apply_quant(const void* x, long long ldx, void* q, long long ldq, float* scale, unsigned int* amax_ws,
                                           int B, int HW, int C, int groups, const double* sums, const float* gamma,
                                           const float* beta, float eps, int silu, void* stream) {
    const char* who = "supir_groupnorm_apply_quant";
    const auto al = [](const void* p, int b) { return (reinterpret_cast<uintptr_t>(p) & (b - 1)) == 0; };
    SUPIR_REQUIRE(x && q && scale && amax_ws && sums, "%s: null pointer", who);
    SUPIR_REQUIRE(B > 0 && HW > 0, "%s: bad shape B=%d HW=%d", who, B, HW);
    SUPIR_REQUIRE(groups > 0 && C % 16 == 0 && C % groups == 0 && C <= 8192 && ldx % 8 == 0 && ldx >= C && ldq % 16 == 0 && ldq >= C,
                  "%s: unsupported C=%d groups=%d ldx=%lld ldq=%lld (C, ldq multiples of 16, ldx of 8)", who, C, groups, ldx, ldq);
    SUPIR_REQUIRE(al(x, 16) && al(q, 16) && al(scale, 4) && al(amax_ws, 4), "%s: misaligned pointer (x, q: 16 bytes; scale, amax_ws: 4)",
                  who);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int cvc = C >> 3;
    int kp = 512 / cvc;
    if (kp < 1) kp = 1;
    const int threads = kp * cvc;
    int ppb = kp * 32;
    if (ppb > HW) ppb = (HW + kp - 1) / kp * kp;
    const int bx = (HW + ppb - 1) / ppb;
    const double count = (double)HW * (C / groups);
    const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
    // the accumulator is reset on the stream (a memset node inside a captured graph), never by the host
    SUPIR_CHECK_CUDA(cudaMemsetAsync(amax_ws, 0, sizeof(unsigned int) * B, st));
    gn_amax_kernel<<<dim3(bx, B), (threads + 31) / 32 * 32, 0, st>>>(xp, ldx, HW, C, groups, sums, count, gamma, beta, eps, silu, ppb,
                                                                      amax_ws);
    gn_apply_quant_kernel<<<dim3(bx, B), threads, 0, st>>>(xp, ldx, reinterpret_cast<uint8_t*>(q), ldq, scale, amax_ws, HW, C, groups,
                                                           sums, count, gamma, beta, eps, silu, ppb);
    count_launch(2);
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

template <class E>
static int zerosft_apply_impl(const char* who, const void* h, long long ldh, const void* skip_raw, long long lds, int C1,
                              const void* gamma_beta, long long ldgb, void* out, long long ldo, int B, int HW, int C, int groups,
                              const double* sums, const float* gn_weight, const float* gn_bias, float eps,
                              const float* control_scale, void* stream) {
    SUPIR_REQUIRE(h && gamma_beta && out && sums && gn_weight && gn_bias && control_scale, "%s: null pointer", who);
    SUPIR_REQUIRE(C % 8 == 0 && C1 % 8 == 0 && C % groups == 0 && (C1 == C || skip_raw), "%s: bad channels", who);
    SUPIR_REQUIRE(C <= 8192, "%s: C=%d too large", who, C);
    const int cvc = C >> 3;
    int kp = 512 / cvc;
    if (kp < 1) kp = 1;
    int ppb = kp * 16;
    if (ppb > HW) ppb = (HW + kp - 1) / kp * kp;
    const int bx = (HW + ppb - 1) / ppb;
    using T = typename E::T;
    sft_apply_kernel<E><<<dim3(bx, B), kp * cvc, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const T*>(h), ldh, reinterpret_cast<const T*>(skip_raw), lds, C1,
        reinterpret_cast<const T*>(gamma_beta), ldgb, reinterpret_cast<T*>(out), ldo, HW, C,
        groups, sums, (double)HW * (C / groups), gn_weight, gn_bias, eps, control_scale, ppb);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_zerosft_apply(const void* h, long long ldh, const void* skip_raw, long long lds, int C1,
                                   const void* gamma_beta, long long ldgb, void* out, long long ldo, int B, int HW,
                                   int C, int groups, const double* sums, const float* gn_weight, const float* gn_bias,
                                   float eps, const float* control_scale, void* stream) {
    return zerosft_apply_impl<Bf16>("supir_zerosft_apply", h, ldh, skip_raw, lds, C1, gamma_beta, ldgb, out, ldo, B, HW, C, groups,
                                    sums, gn_weight, gn_bias, eps, control_scale, stream);
}

extern "C" int supir_zerosft_apply_f16(const void* h, long long ldh, const void* skip_raw, long long lds, int C1,
                                       const void* gamma_beta, long long ldgb, void* out, long long ldo, int B, int HW,
                                       int C, int groups, const double* sums, const float* gn_weight, const float* gn_bias,
                                       float eps, const float* control_scale, void* stream) {
    return zerosft_apply_impl<F16>("supir_zerosft_apply_f16", h, ldh, skip_raw, lds, C1, gamma_beta, ldgb, out, ldo, B, HW, C, groups,
                                   sums, gn_weight, gn_bias, eps, control_scale, stream);
}

template <class E, bool QUANT = false>
static int launch_layernorm(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, const float* gamma,
                            const float* beta, float eps, float2* stats, void* stream, uint8_t* q = nullptr, long long ldq = 0,
                            float* qscale = nullptr);

extern "C" int supir_layernorm_stats(const void* x, long long ldx, long long rows, int C, float eps, float* stats, void* stream) {
    SUPIR_REQUIRE(x && stats && rows > 0, "supir_layernorm_stats: bad args");
    SUPIR_REQUIRE(C % 8 == 0 && C <= 2048 && ldx % 8 == 0, "supir_layernorm_stats: unsupported C=%d", C);
    SUPIR_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 7) == 0, "supir_layernorm_stats: stats must be 8-byte aligned");
    return launch_layernorm<Bf16>(x, ldx, nullptr, 0, rows, C, nullptr, nullptr, eps, reinterpret_cast<float2*>(stats), stream);
}

extern "C" int supir_layernorm_stats_f16(const void* x, long long ldx, long long rows, int C, float eps, float* stats, void* stream) {
    SUPIR_REQUIRE(x && stats && rows > 0, "supir_layernorm_stats_f16: bad args");
    SUPIR_REQUIRE(C % 8 == 0 && C <= 2048 && ldx % 8 == 0, "supir_layernorm_stats_f16: unsupported C=%d", C);
    SUPIR_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 7) == 0, "supir_layernorm_stats_f16: stats must be 8-byte aligned");
    return launch_layernorm<F16>(x, ldx, nullptr, 0, rows, C, nullptr, nullptr, eps, reinterpret_cast<float2*>(stats), stream);
}

extern "C" int supir_layernorm_bf16(const void* x, long long ldx, void* y, long long ldy, long long rows, int C,
                                    const float* gamma, const float* beta, float eps, void* stream) {
    SUPIR_REQUIRE(x && y && gamma && beta, "supir_layernorm_bf16: null pointer");
    SUPIR_REQUIRE(C % 8 == 0 && C <= 2048 && ldx % 8 == 0 && ldy % 8 == 0, "supir_layernorm_bf16: unsupported C=%d", C);
    return launch_layernorm<Bf16>(x, ldx, y, ldy, rows, C, gamma, beta, eps, nullptr, stream);
}

extern "C" int supir_layernorm_f16(const void* x, long long ldx, void* y, long long ldy, long long rows, int C,
                                   const float* gamma, const float* beta, float eps, void* stream) {
    SUPIR_REQUIRE(x && y && gamma && beta, "supir_layernorm_f16: null pointer");
    SUPIR_REQUIRE(C % 8 == 0 && C <= 2048 && ldx % 8 == 0 && ldy % 8 == 0, "supir_layernorm_f16: unsupported C=%d", C);
    return launch_layernorm<F16>(x, ldx, y, ldy, rows, C, gamma, beta, eps, nullptr, stream);
}

extern "C" int supir_layernorm_quant(const void* x, long long ldx, void* q, long long ldq, float* scale, long long rows, int C,
                                     const float* gamma, const float* beta, float eps, void* stream) {
    SUPIR_REQUIRE(x && q && scale && gamma && beta, "supir_layernorm_quant: null pointer");
    SUPIR_REQUIRE(rows > 0, "supir_layernorm_quant: bad rows %lld", rows);
    SUPIR_REQUIRE(C % 16 == 0 && C <= 2048 && ldx % 8 == 0 && ldq % 16 == 0 && ldq >= C && ldx >= C,
                  "supir_layernorm_quant: unsupported C=%d ldx=%lld ldq=%lld (C, ldq multiples of 16, C <= 2048)", C, ldx, ldq);
    SUPIR_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(scale) & 3) == 0 && (reinterpret_cast<uintptr_t>(gamma) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(beta) & 15) == 0,
                  "supir_layernorm_quant: misaligned pointer (x, q, gamma, beta: 16 bytes; scale: 4)");
    return launch_layernorm<Bf16, true>(x, ldx, nullptr, 0, rows, C, gamma, beta, eps, nullptr, stream,
                                        reinterpret_cast<uint8_t*>(q), ldq, scale);
}

template <class E, bool QUANT>
static int launch_layernorm(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, const float* gamma,
                            const float* beta, float eps, float2* stats, void* stream, uint8_t* q, long long ldq, float* qscale) {
    const int warps = 8;
    long long blocks = (rows + warps - 1) / warps;
    const long long cap = (long long)device_sm_count() * 16;       // a few resident waves; warps then loop over rows
    if (blocks > cap) blocks = cap;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const typename E::T* xp = reinterpret_cast<const typename E::T*>(x);
    typename E::T* yp = reinterpret_cast<typename E::T*>(y);
    const int nv = C >> 3;
    if (nv <= 96)
        layernorm_kernel<3, E, QUANT><<<(unsigned)blocks, warps * 32, 0, st>>>(xp, ldx, yp, ldy, rows, C, gamma, beta, eps, stats, q, ldq, qscale);
    else if (nv <= 160)
        layernorm_kernel<5, E, QUANT><<<(unsigned)blocks, warps * 32, 0, st>>>(xp, ldx, yp, ldy, rows, C, gamma, beta, eps, stats, q, ldq, qscale);
    else
        layernorm_kernel<8, E, QUANT><<<(unsigned)blocks, warps * 32, 0, st>>>(xp, ldx, yp, ldy, rows, C, gamma, beta, eps, stats, q, ldq, qscale);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_softmax_rows(const float* S, long long lds, void* P, long long ldp, long long rows, int cols,
                                  float scale, void* stream) {
    SUPIR_REQUIRE(S && P && rows > 0 && cols > 0, "supir_softmax_rows: bad args");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t smem = (size_t)((cols + 7) / 8 * 8) * sizeof(float);
    const bool aligned = (lds % 4 == 0) && (ldp % 8 == 0) && (reinterpret_cast<uintptr_t>(S) % 16 == 0) &&
                         (reinterpret_cast<uintptr_t>(P) % 16 == 0);
    if (aligned && cols >= 1024 && smem <= 200 * 1024) {
        static size_t max_set_dev[64] = {};
    size_t& max_set = max_set_dev[current_device_slot()];
        if (smem > 48 * 1024 && smem > max_set) {
            SUPIR_CHECK_CUDA(cudaFuncSetAttribute(softmax_rows_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            max_set = smem;
        }
        softmax_rows_smem_kernel<<<(unsigned)rows, 1024, smem, st>>>(S, lds, reinterpret_cast<__nv_bfloat16*>(P), ldp, cols, scale);
    } else {
        softmax_rows_kernel<<<(unsigned)rows, 256, 0, st>>>(S, lds, reinterpret_cast<__nv_bfloat16*>(P), ldp, cols, scale);
    }
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}
