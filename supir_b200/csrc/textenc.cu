// supir_b200 — kernels of the text conditioner (SURVEY.md §8(f)2): the CLIP-L and OpenCLIP bigG text towers run ONCE per
// image on 77 tokens (sgm/modules/encoders/modules.py:484-507, 553-609), so nothing here is throughput-critical: the
// projections go through the wgmma GEMM of gemm.cu, and the pieces that GEMM does not cover are these small CUDA-core
// kernels — token / position embedding gather, LayerNorm on the fp32 residual stream (the reference keeps that stream in fp32:
// autocast only lowers the matmuls), causal attention over <= 128 tokens, and the MLP activations (quick-GELU for CLIP-L,
// exact GELU for bigG).
#include "common.cuh"
#include "supir_b200.h"

namespace supir {

static inline unsigned te_blocks_for(long long n, int threads) {
    long long b = (n + threads - 1) / threads;
    const long long cap = device_sm_count() * 16LL;   // grid-stride loops: 16 blocks per SM
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (unsigned)b;
}

// out[r, :] = table[idx[r], :] (+ pos[r % L, :]); fp32, C % 4 == 0. Indices outside [0, table_rows) are clamped.
// nn.Embedding lookups + positional add (HF CLIPTextEmbeddings; open_clip `token_embedding(text) + positional_embedding`,
// modules.py:569-570), and the EOT-row gather of `pool` (modules.py:584-590).
__global__ void gather_rows_f32_kernel(const float* __restrict__ table, long long ldt, int table_rows, const int* __restrict__ idx,
                                       const float* __restrict__ pos, long long ldp, int L, float* __restrict__ out, long long ldo,
                                       long long rows, int C) {
    const int cv = C >> 2;
    const long long total = rows * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cv;
        const int c = (int)(i % cv);
        int t = __ldg(idx + r);
        t = t < 0 ? 0 : (t >= table_rows ? table_rows - 1 : t);
        float4 v = __ldg(reinterpret_cast<const float4*>(table + (long long)t * ldt + c * 4));
        if (pos) {
            const float4 p = __ldg(reinterpret_cast<const float4*>(pos + (r % L) * ldp + c * 4));
            v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
        }
        *reinterpret_cast<float4*>(out + r * ldo + c * 4) = v;
    }
}

// LayerNorm of fp32 rows (two-pass: mean, then the variance about it, like ATen), one warp per row; writes bf16 (the next
// GEMM's operand) and / or fp32 (ln_final feeding the pooled projection, `last` layer outputs).
__global__ void layernorm_f32_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ yb, long long ldyb,
                                     float* __restrict__ yf, long long ldyf, long long rows, int C, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float eps) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    for (long long r = (long long)blockIdx.x * warps + warp; r < rows; r += (long long)gridDim.x * warps) {
        const float* xr = x + r * ldx;
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s += xr[c];
        const float mean = warp_sum(s) / (float)C;
        float q = 0.f;
        for (int c = lane; c < C; c += 32) {
            const float d = xr[c] - mean;
            q = fmaf(d, d, q);
        }
        const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
        for (int c = lane; c < C; c += 32) {
            const float v = (xr[c] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c);
            if (yb) yb[r * ldyb + c] = __float2bfloat16_rn(v);
            if (yf) yf[r * ldyf + c] = v;
        }
    }
}

// Attention over a short sequence (L <= 128 tokens, head_dim 64) with an optional causal mask — the text towers' self-attention
// (HF CLIPAttention with the causal mask; open_clip nn.MultiheadAttention with attn_mask, modules.py:571). One CTA per
// (batch, head): K (rows padded to 33 words: conflict-free when every lane reads another key) and V in shared memory as bf16,
// one warp per query row: lanes own keys for the scores and the softmax, then own two output columns each for P V.
constexpr int TE_LMAX = 128;
constexpr int TE_WARPS = 8;
__global__ void __launch_bounds__(TE_WARPS * 32)
attention_small_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ k, long long ldk,
                       const __nv_bfloat16* __restrict__ v, long long ldv, __nv_bfloat16* __restrict__ out, long long ldo, int H,
                       int L, float scale, int causal) {
    __shared__ uint32_t Ks[TE_LMAX * 33];
    __shared__ uint32_t Vs[TE_LMAX * 32];
    __shared__ float qs[TE_WARPS][64];
    __shared__ float ps[TE_WARPS][TE_LMAX];
    const int b = blockIdx.x / H, h = blockIdx.x % H;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < L * 32; i += blockDim.x) {
        const int j = i >> 5, w = i & 31;
        Ks[j * 33 + w] = *reinterpret_cast<const uint32_t*>(k + ((long long)b * L + j) * ldk + h * 64 + 2 * w);
        Vs[j * 32 + w] = *reinterpret_cast<const uint32_t*>(v + ((long long)b * L + j) * ldv + h * 64 + 2 * w);
    }
    __syncthreads();
    for (int i = warp; i < L; i += TE_WARPS) {
        const float2 qf = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(q + ((long long)b * L + i) * ldq + h * 64 + 2 * lane));
        qs[warp][2 * lane] = qf.x * scale;
        qs[warp][2 * lane + 1] = qf.y * scale;
        __syncwarp();
        const int n = causal ? i + 1 : L;
        float s[4];
        float m = -INFINITY;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int j = lane + 32 * t;
            s[t] = -INFINITY;
            if (j < n) {
                float acc = 0.f;
#pragma unroll 8
                for (int w = 0; w < 32; ++w) {
                    const float2 kf = unpack_bf16x2(Ks[j * 33 + w]);
                    acc = fmaf(qs[warp][2 * w], kf.x, acc);
                    acc = fmaf(qs[warp][2 * w + 1], kf.y, acc);
                }
                s[t] = acc;
            }
            m = fmaxf(m, s[t]);
        }
        m = warp_max(m);
        float sum = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int j = lane + 32 * t;
            const float p = (j < n) ? __expf(s[t] - m) : 0.f;
            sum += p;
            ps[warp][j] = p;
        }
        const float inv = 1.0f / warp_sum(sum);
        __syncwarp();
        float o0 = 0.f, o1 = 0.f;
        for (int j = 0; j < n; ++j) {
            const float p = ps[warp][j];
            const float2 vf = unpack_bf16x2(Vs[j * 32 + lane]);
            o0 = fmaf(p, vf.x, o0);
            o1 = fmaf(p, vf.y, o1);
        }
        *reinterpret_cast<uint32_t*>(out + ((long long)b * L + i) * ldo + h * 64 + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
        __syncwarp();
    }
}

// y = act(x) on bf16 rows: mode 0 = exact (erf) GELU — open_clip's nn.GELU; mode 1 = quick-GELU x * sigmoid(1.702 x) — the
// `quick_gelu` of openai/clip-vit-large-patch14. x and y may alias.
__global__ void activation_bf16_kernel(const __nv_bfloat16* x, long long ldx, __nv_bfloat16* y, long long ldy, long long rows,
                                       int cols, int mode) {
    const int cv = cols >> 3;
    const long long total = rows * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cv;
        const int c = (int)(i % cv);
        const uint4 u = *reinterpret_cast<const uint4*>(x + r * ldx + c * 8);
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
        uint32_t o[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = unpack_bf16x2(w[t]);
            float a, bq;
            if (mode == 0) {
                a = gelu_erf_f(f.x);
                bq = gelu_erf_f(f.y);
            } else {
                a = __fdividef(f.x, 1.0f + __expf(-1.702f * f.x));
                bq = __fdividef(f.y, 1.0f + __expf(-1.702f * f.y));
            }
            o[t] = pack_bf16x2(a, bq);
        }
        *reinterpret_cast<uint4*>(y + r * ldy + c * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

}  // namespace supir

using namespace supir;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)
#define DONE()                              \
    do {                                    \
        count_launch();                     \
        SUPIR_CHECK_CUDA(cudaGetLastError()); \
        return SUPIR_OK;                    \
    } while (0)

extern "C" int supir_gather_rows_f32(const float* table, long long ldt, int table_rows, const int* idx, const float* pos,
                                     long long ldp, int L, float* out, long long ldo, long long rows, int C, void* stream) {
    SUPIR_REQUIRE(table && idx && out && rows > 0 && table_rows > 0, "supir_gather_rows_f32: bad args");
    SUPIR_REQUIRE(C > 0 && C % 4 == 0 && ldt % 4 == 0 && ldo % 4 == 0 && ldt >= C && ldo >= C, "supir_gather_rows_f32: C / leading dims must be multiples of 4");
    SUPIR_REQUIRE(!pos || (L > 0 && ldp % 4 == 0 && ldp >= C), "supir_gather_rows_f32: bad positional table");
    SUPIR_REQUIRE(((reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(pos)) & 15) == 0,
                  "supir_gather_rows_f32: pointers must be 16-byte aligned");
    gather_rows_f32_kernel<<<te_blocks_for(rows * (C >> 2), 256), 256, 0, ST(stream)>>>(table, ldt, table_rows, idx, pos, ldp,
                                                                                         L > 0 ? L : 1, out, ldo, rows, C);
    DONE();
}

extern "C" int supir_layernorm_f32(const float* x, long long ldx, void* y_bf16, long long ldyb, float* y_f32, long long ldyf,
                                   long long rows, int C, const float* gamma, const float* beta, float eps, void* stream) {
    SUPIR_REQUIRE(x && gamma && beta && (y_bf16 || y_f32) && rows > 0 && C > 0, "supir_layernorm_f32: bad args");
    SUPIR_REQUIRE(ldx >= C && (!y_bf16 || ldyb >= C) && (!y_f32 || ldyf >= C), "supir_layernorm_f32: leading dims smaller than C");
    const int warps = 8;
    long long blocks = (rows + warps - 1) / warps;
    if (blocks > device_sm_count() * 8LL) blocks = device_sm_count() * 8LL;
    layernorm_f32_kernel<<<(unsigned)blocks, warps * 32, 0, ST(stream)>>>(x, ldx, BF(y_bf16), ldyb, y_f32, ldyf, rows, C, gamma, beta, eps);
    DONE();
}

extern "C" int supir_attention_small_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                                          void* out, long long ldo, int B, int H, int L, int head_dim, float scale, int causal,
                                          void* stream) {
    SUPIR_REQUIRE(q && k && v && out && B > 0 && H > 0, "supir_attention_small_bf16: bad args");
    SUPIR_REQUIRE(head_dim == 64, "supir_attention_small_bf16: head_dim %d unsupported (64 only)", head_dim);
    SUPIR_REQUIRE(L >= 1 && L <= TE_LMAX, "supir_attention_small_bf16: %d tokens (1..%d supported)", L, TE_LMAX);
    SUPIR_REQUIRE(ldq % 2 == 0 && ldk % 2 == 0 && ldv % 2 == 0 && ldo % 2 == 0 && ldq >= H * 64 && ldk >= H * 64 && ldv >= H * 64 && ldo >= H * 64,
                  "supir_attention_small_bf16: bad leading dims");
    SUPIR_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                    reinterpret_cast<uintptr_t>(out)) & 3) == 0, "supir_attention_small_bf16: pointers must be 4-byte aligned");
    attention_small_kernel<<<(unsigned)(B * H), TE_WARPS * 32, 0, ST(stream)>>>(CBF(q), ldq, CBF(k), ldk, CBF(v), ldv, BF(out), ldo, H,
                                                                                 L, scale, causal ? 1 : 0);
    DONE();
}

extern "C" int supir_activation_bf16(const void* x, long long ldx, void* y, long long ldy, long long rows, int cols, int mode,
                                     void* stream) {
    SUPIR_REQUIRE(x && y && rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= cols && ldy >= cols,
                  "supir_activation_bf16: bad args");
    SUPIR_REQUIRE(mode == 0 || mode == 1, "supir_activation_bf16: mode %d not in {0 (GELU), 1 (quick-GELU)}", mode);
    SUPIR_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "supir_activation_bf16: pointers must be 16-byte aligned");
    activation_bf16_kernel<<<te_blocks_for(rows * (cols >> 3), 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, rows, cols, mode);
    DONE();
}
