// supir_b200 — FP8 attention (the fp8_attention option of the FP8 mode): softmax(Q K^T / sqrt(64)) V on e4m3 tensor cores for
// the UNet's self-attention and ZeroCrossAttn, head_dim 64.
//
// Quantization points (DESIGN.md §7). With s = amax / 448 and code = RNE(x * (448 / amax)) (e4m3_row_scale; scale 1 when
// amax = 0), every scale inside one image:
//   Q  one scale per (token, head) over its 64 channels            sq [B*Lq, H]
//   K  one scale per (image, head) over all Lk tokens x 64 channels sk [B, H]
//   V  one scale per (image, head, channel) over all Lk tokens      sv [B, H, 64]
//   P  the fixed power of two 2^8: code = RNE_satfinite(2^8 p), p = 2^(logit - running max) <= 1 in fp32
// The row sum l adds the unrounded fp32 p (as the 16-bit kernels do); O[q, d] = acc[q, d] * sv[d] / (2^8 l), rounded once to bf16.
//
// supir_attention_quant_fp8 writes the operands from bf16 q, k, v (column slices of the fused QKV buffer, or separate q and kv):
// an amax pass over K and V into an unsigned workspace (atomicMax on the bits of non-negative floats: order-independent, so
// deterministic), then the quantize passes. V is written transposed, vt8 [B, H, 64, ld_vt], because e4m3 wgmma takes K-major
// operands only and the contraction of P V runs over keys. Inside every group of 32 keys vt8's key order is permuted so that P
// goes from the Q K^T accumulator fragment straight into the m64k32 A fragment: k position kappa = 16 a + 4 c + i carries key
// 16 a + 2 c + (i & 1) + 8 (i >> 1). Positions from Lk up to ld_vt hold zeros.
//
// supir_attention_fp8: attention_wgmma_kernel's structure with e4m3 operands. 384 threads; warpgroup 0's thread 0 is the TMA
// producer (Q once, then K(j) and Vt(j) of every 128-key block through a ring); warpgroups 1, 2 own 64 query rows each:
//   S = Q K^T   two m64n128k32 steps, Q and K 64-byte rows with 64-byte swizzle
//   softmax     per-row logit scale sq[row] * sk * scale * log2e, running max, P = 2^(x - m) (MUFU or ex2_emulated, split
//               fixed by ATT_FP8_EMU), l += P, A registers = cvt.rn.satfinite.e4m3x2 of 2^8 P
//   O += P Vt   four m64n64k32 steps into a per-block accumulator, A from registers, B = the Vt tile (128-byte rows,
//               128-byte swizzle); O = alpha O + block in fp32
// supir_set_attention_exp_emulation / supir_set_attention_alu_pack do not affect this kernel.
#include "common.cuh"
#include "supir_b200.h"
#include "wgmma.cuh"

namespace supir {

// exponential pairs of every 4 taken from ex2_emulated (the FMA-pipe polynomial) instead of MUFU.EX2. Measured on an H100 80GB
// HBM3 at 700 W (DESIGN.md §8), 0 is the fastest at every SUPIR shape: 1, 2 and 3 of 4 emulated cost 5-11 %, 3-9 % and 15-22 %.
static constexpr int ATT_FP8_EMU = 0;

static constexpr int AF8_BM = 128, AF8_BKV = 128, AF8_THREADS = 384;
static constexpr int AF8_TILE = 128 * 64;          // 8 KB: Q (128 rows x 64 B), K (128 keys x 64 B) or Vt (64 channels x 128 keys)
static constexpr int AF8_SLOTS = 6;
static constexpr int AF8_OFF_RING = AF8_TILE;
static constexpr int AF8_OFF_BAR = AF8_OFF_RING + AF8_SLOTS * AF8_TILE;
static constexpr int AF8_SMEM = AF8_OFF_BAR + 256 + 1024;
static constexpr float AF8_P_SCALE = 256.f;        // 2^8

struct AttnFp8Params {
    int Lq, Lk, H;
    long long ldo;
    __nv_bfloat16* out;
    const float* sq;
    const float* sk;
    const float* sv;
    float scale_log2;
};

__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
    return __nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, __NV_E4M3);   // cvt.rn.satfinite.e4m3x2.f32
}

__global__ void __launch_bounds__(AF8_THREADS, 1)
attention_fp8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnFp8Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* ring = smem + AF8_OFF_RING;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AF8_OFF_BAR);
    uint64_t* q_full = bars;
    uint64_t* slot_full = bars + 1;
    uint64_t* slot_empty = slot_full + AF8_SLOTS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AF8_BM, head = blockIdx.y, batch = blockIdx.z;
    const int nblk = (p.Lk + AF8_BKV - 1) / AF8_BKV;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        mbar_init(q_full, 1);
        for (int s = 0; s < AF8_SLOTS; ++s) { mbar_init(&slot_full[s], 1); mbar_init(&slot_empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            mbar_expect_tx(q_full, AF8_TILE);
            tma_load_2d(sQ, &tmQ, q_full, head * 64, batch * p.Lq + q0);
            int slot = 0;
            uint32_t phase = 0;
            auto push = [&](const CUtensorMap* tm, int c0, int c1) {
                mbar_wait(&slot_empty[slot], phase ^ 1);
                mbar_expect_tx(&slot_full[slot], AF8_TILE);
                tma_load_2d(ring + slot * AF8_TILE, tm, &slot_full[slot], c0, c1);
                if (++slot == AF8_SLOTS) { slot = 0; phase ^= 1; }
            };
            for (int j = 0; j < nblk; ++j) {
                push(&tmK, head * 64, batch * p.Lk + j * AF8_BKV);
                push(&tmV, j * AF8_BKV, (batch * p.H + head) * 64);
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int wg = (warp - 4) >> 2;
        const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // fragment rows r_lo and r_lo + 8
        const int cq = 2 * (lane & 3);
        const float sk = p.sk[batch * p.H + head];
        float sl2[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int qrow = q0 + r_lo + 8 * h;            // rows past Lq are computed from the next rows' codes, never stored
            const float sq = qrow < p.Lq ? p.sq[((long long)batch * p.Lq + qrow) * p.H + head] : 1.f;
            sl2[h] = sq * sk * p.scale_log2;
        }
        int slot = 0;
        uint32_t phase = 0;
        float o[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        mbar_wait(q_full, 0);
        for (int j = 0; j < nblk; ++j) {
            // ---- S = Q K_j^T (codes) ----
            float s[64];
            mbar_wait(&slot_full[slot], phase);
            wgmma_fence();
            {
                const uint32_t qa = smem_u32(sQ + wg * 64 * 64);
                const uint32_t ka = smem_u32(ring + slot * AF8_TILE);
#pragma unroll
                for (int kk = 0; kk < 2; ++kk)
                    wgmma_ss_n128<E4m3>(s, wgmma_desc_sw64(qa + 32 * kk), wgmma_desc_sw64(ka + 32 * kk), kk);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_operands(s);
            __syncwarp();
            if (lane == 0) mbar_arrive(&slot_empty[slot]);
            if (++slot == AF8_SLOTS) { slot = 0; phase ^= 1; }

            // ---- online softmax: element 4 t + 2 h + e = row r_lo + 8 h, key 8 t + cq + e ----
            const int kv_valid = min(AF8_BKV, p.Lk - j * AF8_BKV);
            if (kv_valid < AF8_BKV) {
#pragma unroll
                for (int t = 0; t < 16; ++t)
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (8 * t + cq + (e & 1) >= kv_valid) s[4 * t + e] = -INFINITY;
            }
            float alpha[2], negm[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float mx = -INFINITY;
#pragma unroll
                for (int t = 0; t < 16; ++t) mx = fmaxf(mx, fmaxf(s[4 * t + 2 * h], s[4 * t + 2 * h + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[h], mx * sl2[h]);      // every block holds >= 1 valid key: finite
                alpha[h] = ex2_approx(m_run[h] - m_new);
                m_run[h] = m_new;
                negm[h] = -m_new;
                l_run[h] *= alpha[h];
            }
            // P as m64k32 A fragments, one per 32 keys: t = 4 g + u holds keys 32 g + 8 u + {cq, cq + 1}; register (u >> 1) * 2 + h
            // takes u = 0, 1 (or 2, 3) as its low / high 16 bits, i.e. k positions 4c..4c+3 carry keys 2c, 2c+1, 8+2c, 9+2c
            uint32_t pa[4][4];
#pragma unroll
            for (int g = 0; g < 4; ++g) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    uint32_t half[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int t = 4 * g + u;
                        const float x0 = fmaf(s[4 * t + 2 * h], sl2[h], negm[h]);
                        const float x1 = fmaf(s[4 * t + 2 * h + 1], sl2[h], negm[h]);
                        const int q = (2 * t + h) & 3;
                        constexpr int EMU = ATT_FP8_EMU;
                        const bool emulate = (EMU == 4) || (EMU == 3 && q != 1) || (EMU == 2 && (q & 1)) || (EMU == 1 && q == 3);
                        const float e0 = emulate ? ex2_emulated(x0) : ex2_approx(x0);
                        const float e1 = emulate ? ex2_emulated(x1) : ex2_approx(x1);
                        l_run[h] += e0 + e1;
                        half[u] = e4m3x2(e0 * AF8_P_SCALE, e1 * AF8_P_SCALE);
                    }
                    pa[g][h] = __byte_perm(half[0], half[1], 0x5410);
                    pa[g][2 + h] = __byte_perm(half[2], half[3], 0x5410);
                }
            }

            // ---- O = alpha O + P Vt_j: the block's product in its own accumulator (e4m3 wgmma adds with reduced alignment
            // precision, so its chain stays four k-steps long), merged into O with one fp32 fma ----
            float ob[32];
            mbar_wait(&slot_full[slot], phase);
            wgmma_fence();
            {
                const uint32_t va = smem_u32(ring + slot * AF8_TILE);
#pragma unroll
                for (int g = 0; g < 4; ++g) wgmma_rs_n64_e4m3(ob, pa[g], wgmma_desc_sw128(va + 32 * g), g);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_operands(ob);
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = fmaf(o[i], alpha[(i >> 1) & 1], ob[i]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&slot_empty[slot]);
            if (++slot == AF8_SLOTS) { slot = 0; phase ^= 1; }
        }

        // ---- O * sv / (2^8 l) -> bf16 ----
        const float* sv = p.sv + ((long long)batch * p.H + head) * 64 + cq;
        float svr[16];
#pragma unroll
        for (int t = 0; t < 8; ++t) { svr[2 * t] = sv[8 * t]; svr[2 * t + 1] = sv[8 * t + 1]; }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float l = l_run[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = 1.f / (l * AF8_P_SCALE);
            const int qrow = q0 + r_lo + 8 * h;
            if (qrow < p.Lq) {
                __nv_bfloat16* dst = p.out + ((long long)batch * p.Lq + qrow) * p.ldo + head * 64 + cq;
#pragma unroll
                for (int t = 0; t < 8; ++t)
                    *reinterpret_cast<uint32_t*>(dst + 8 * t) =
                        pack_bf16x2(o[4 * t + 2 * h] * svr[2 * t] * inv, o[4 * t + 2 * h + 1] * svr[2 * t + 1] * inv);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// operand pass
// ---------------------------------------------------------------------------------------------
static constexpr int AQ_TOK = 64;        // keys per block of the amax pass
static constexpr int AQ_ROWS = 16;       // rows per block of the Q / K quantize pass

__device__ __forceinline__ void unpack8(const uint4 u, float (&f)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const float2 x = unpack_bf16x2(w[t]);
        f[2 * t] = x.x;
        f[2 * t + 1] = x.y;
    }
}

// amax_k[b * H + h] over K, amax_v[(b * H + h) * 64 + d] over V. Thread t owns channels 8t..8t+7 (8 threads per head).
__global__ void attn_kv_amax_kernel(const __nv_bfloat16* __restrict__ k, long long ldk, const __nv_bfloat16* __restrict__ v,
                                    long long ldv, int H, int Lk, unsigned int* __restrict__ amax_k, unsigned int* __restrict__ amax_v) {
    const int t = threadIdx.x, b = blockIdx.y;
    const bool active = t < H * 8;
    const int j0 = blockIdx.x * AQ_TOK, j1 = min(j0 + AQ_TOK, Lk);
    float mk = 0.f, mv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (active) {
        for (int j = j0; j < j1; ++j) {
            const long long row = (long long)b * Lk + j;
            float fk[8], fv[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(k + row * ldk + 8 * t)), fk);
            unpack8(__ldg(reinterpret_cast<const uint4*>(v + row * ldv + 8 * t)), fv);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                mk = fmaxf(mk, fabsf(fk[i]));
                mv[i] = fmaxf(mv[i], fabsf(fv[i]));
            }
        }
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) mk = fmaxf(mk, __shfl_xor_sync(0xffffffffu, mk, o));
    if (!active) return;
    if ((t & 7) == 0) atomicMax(amax_k + b * H + (t >> 3), __float_as_uint(mk));
#pragma unroll
    for (int i = 0; i < 8; ++i) atomicMax(amax_v + ((long long)b * H * 64) + 8 * t + i, __float_as_uint(mv[i]));
}

// Q rows (blocks [0, nbq)): row amax per head over the 8 threads of the head, codes and sq. K rows (blocks from nbq): codes
// with the (image, head) scale of amax_k.
__global__ void attn_qk_quant_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ k,
                                     long long ldk, uint8_t* __restrict__ q8, long long ldq8, float* __restrict__ sq,
                                     uint8_t* __restrict__ k8, long long ldk8, const unsigned int* __restrict__ amax_k, int H,
                                     int Lk, long long rows_q, long long rows_k, int nbq) {
    const int t = threadIdx.x;
    const bool active = t < H * 8;
    const bool is_q = blockIdx.x < nbq;
    const long long r0 = (long long)(is_q ? blockIdx.x : blockIdx.x - nbq) * AQ_ROWS;
    const long long rows = is_q ? rows_q : rows_k;
    for (long long r = r0; r < min(r0 + AQ_ROWS, rows); ++r) {
        float f[8];
        float amax = 0.f;
        if (active) {
            unpack8(__ldg(reinterpret_cast<const uint4*>((is_q ? q + r * ldq : k + r * ldk) + 8 * t)), f);
#pragma unroll
            for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (!active) continue;
        if (!is_q) amax = __uint_as_float(amax_k[(r / Lk) * H + (t >> 3)]);
        float s, inv;
        e4m3_row_scale(amax, s, inv);
        if (is_q && (t & 7) == 0) sq[r * H + (t >> 3)] = s;
        const uint2 c = make_uint2(pack_e4m3x4(f[0] * inv, f[1] * inv, f[2] * inv, f[3] * inv),
                                   pack_e4m3x4(f[4] * inv, f[5] * inv, f[6] * inv, f[7] * inv));
        *reinterpret_cast<uint2*>((is_q ? q8 + r * ldq8 : k8 + r * ldk8) + 8 * t) = c;
    }
}

// vt8 [B, H, 64, ld_vt] from V: one block per (128 key positions, head, image), 256 threads. The 128 keys are quantized with
// the channel scales into shared memory at their permuted positions, then written as 64 rows of 128 bytes. Block x = 0 also
// writes sv and sk.
__global__ void attn_v_quant_kernel(const __nv_bfloat16* __restrict__ v, long long ldv, uint8_t* __restrict__ vt8, long long ld_vt,
                                    float* __restrict__ sv, float* __restrict__ sk, const unsigned int* __restrict__ amax_k,
                                    const unsigned int* __restrict__ amax_v, int H, int Lk) {
    __shared__ __align__(16) uint8_t tile[64][128 + 16];
    __shared__ float inv_d[64];
    const int t = threadIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int p0 = blockIdx.x * 128;
    const long long bh = (long long)b * H + h;
    if (t < 64) {
        float s, inv;
        e4m3_row_scale(__uint_as_float(amax_v[bh * 64 + t]), s, inv);
        inv_d[t] = inv;
        if (blockIdx.x == 0) sv[bh * 64 + t] = s;
    }
    if (blockIdx.x == 0 && t == 64) {
        float s, inv;
        e4m3_row_scale(__uint_as_float(amax_k[bh]), s, inv);
        sk[bh] = s;
    }
    __syncthreads();
    const int cv = t & 7;                    // channels 8 cv .. 8 cv + 7
#pragma unroll
    for (int pass = 0; pass < 4; ++pass) {
        const int u = pass * 32 + (t >> 3);  // key offset inside the block of 128
        const int j = p0 + u;
        float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (j < Lk) unpack8(__ldg(reinterpret_cast<const uint4*>(v + ((long long)b * Lk + j) * ldv + h * 64 + 8 * cv)), f);
        // key offset w inside its group of 32 -> k position 16 a + 4 c + i with key = 16 a + 2 c + (i & 1) + 8 (i >> 1)
        const int w = u & 31, w16 = w & 15;
        const int pos = (u & ~31) + (w & 16) + 4 * ((w16 >> 1) & 3) + 2 * (w16 >> 3) + (w16 & 1);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float x = f[i] * inv_d[8 * cv + i];
            tile[8 * cv + i][pos] = (uint8_t)__nv_cvt_float_to_fp8(x, __NV_SATFINITE, __NV_E4M3);
        }
    }
    __syncthreads();
    uint8_t* dst = vt8 + bh * 64 * ld_vt;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = i * 256 + t;           // 64 rows x 8 chunks of 16 bytes
        const int d = c >> 3, x = (c & 7) * 16;
        if (p0 + x < ld_vt) *reinterpret_cast<uint4*>(dst + d * ld_vt + p0 + x) = *reinterpret_cast<const uint4*>(&tile[d][x]);
    }
}

}  // namespace supir

using namespace supir;

static bool aligned_to(const void* p, int b) { return (reinterpret_cast<uintptr_t>(p) & (b - 1)) == 0; }

extern "C" int supir_attention_quant_fp8(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                                         void* q8, long long ldq8, float* sq, void* k8, long long ldk8, float* sk, void* vt8,
                                         long long ld_vt, float* sv, unsigned int* amax_ws, int B, int H, int Lq, int Lk,
                                         void* stream) {
    const char* who = "supir_attention_quant_fp8";
    SUPIR_REQUIRE(q && k && v && q8 && sq && k8 && sk && vt8 && sv && amax_ws, "%s: null pointer", who);
    SUPIR_REQUIRE(B > 0 && H > 0 && H <= 128 && Lq > 0 && Lk > 0, "%s: bad shape B=%d H=%d Lq=%d Lk=%d (H <= 128)", who, B, H, Lq, Lk);
    const long long cols = (long long)H * 64;
    SUPIR_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldq >= cols && ldk >= cols && ldv >= cols,
                  "%s: bf16 leading dims must be multiples of 8 and >= H * 64 = %lld", who, cols);
    SUPIR_REQUIRE(ldq8 % 16 == 0 && ldk8 % 16 == 0 && ldq8 >= cols && ldk8 >= cols,
                  "%s: e4m3 leading dims must be multiples of 16 and >= H * 64 = %lld", who, cols);
    SUPIR_REQUIRE(ld_vt % 16 == 0 && ld_vt >= Lk, "%s: ld_vt = %lld must be a multiple of 16 and >= Lk = %d", who, ld_vt, Lk);
    SUPIR_REQUIRE(aligned_to(q, 16) && aligned_to(k, 16) && aligned_to(v, 16) && aligned_to(q8, 16) && aligned_to(k8, 16) &&
                      aligned_to(vt8, 16) && aligned_to(sq, 4) && aligned_to(sk, 4) && aligned_to(sv, 4) && aligned_to(amax_ws, 4),
                  "%s: misaligned pointer (q, k, v, q8, k8, vt8: 16 bytes; scales and amax_ws: 4)", who);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned int* amax_k = amax_ws;
    unsigned int* amax_v = amax_ws + (long long)B * H;
    const int threads = (H * 8 + 31) / 32 * 32;
    // the accumulator is reset on the stream (a memset node inside a captured graph), never by the host
    SUPIR_CHECK_CUDA(cudaMemsetAsync(amax_ws, 0, sizeof(unsigned int) * B * H * 65, st));
    attn_kv_amax_kernel<<<dim3((Lk + AQ_TOK - 1) / AQ_TOK, B), threads, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(k), ldk, reinterpret_cast<const __nv_bfloat16*>(v), ldv, H, Lk, amax_k, amax_v);
    const long long rows_q = (long long)B * Lq, rows_k = (long long)B * Lk;
    const int nbq = (int)((rows_q + AQ_ROWS - 1) / AQ_ROWS), nbk = (int)((rows_k + AQ_ROWS - 1) / AQ_ROWS);
    attn_qk_quant_kernel<<<nbq + nbk, threads, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(q), ldq, reinterpret_cast<const __nv_bfloat16*>(k), ldk, reinterpret_cast<uint8_t*>(q8),
        ldq8, sq, reinterpret_cast<uint8_t*>(k8), ldk8, amax_k, H, Lk, rows_q, rows_k, nbq);
    attn_v_quant_kernel<<<dim3((unsigned)((ld_vt + 127) / 128), H, B), 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(v), ldv, reinterpret_cast<uint8_t*>(vt8), ld_vt, sv, sk, amax_k, amax_v, H, Lk);
    count_launch(3);
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

extern "C" int supir_attention_fp8(const void* q8, long long ldq, const float* sq, const void* k8, long long ldk, const float* sk,
                                   const void* vt8, long long ld_vt, const float* sv, void* out, long long ldo, int B, int H, int Lq,
                                   int Lk, int head_dim, float scale, void* stream) {
    const char* who = "supir_attention_fp8";
    SUPIR_REQUIRE(q8 && sq && k8 && sk && vt8 && sv && out, "%s: null pointer", who);
    SUPIR_REQUIRE(head_dim == 64, "%s: head_dim %d unsupported (64 only)", who, head_dim);
    SUPIR_REQUIRE(B > 0 && H > 0 && H <= 65535 && Lq > 0 && Lk > 0, "%s: bad shape", who);
    SUPIR_REQUIRE(scale > 0.f, "%s: scale must be positive", who);
    const long long cols = (long long)H * 64;
    SUPIR_REQUIRE(ldq % 16 == 0 && ldk % 16 == 0 && ldq >= cols && ldk >= cols,
                  "%s: e4m3 leading dims must be multiples of 16 and >= H * 64 = %lld", who, cols);
    SUPIR_REQUIRE(ld_vt % 16 == 0 && ld_vt >= Lk, "%s: ld_vt = %lld must be a multiple of 16 and >= Lk = %d", who, ld_vt, Lk);
    SUPIR_REQUIRE(ldo % 8 == 0 && ldo >= cols, "%s: ldo must be a multiple of 8 and >= H * 64 = %lld", who, cols);
    // the final store writes two outputs as one 32-bit word
    SUPIR_REQUIRE(aligned_to(q8, 16) && aligned_to(k8, 16) && aligned_to(vt8, 16), "%s: q8, k8, vt8 must be 16-byte aligned", who);
    SUPIR_REQUIRE(aligned_to(out, 4) && aligned_to(sq, 4) && aligned_to(sk, 4) && aligned_to(sv, 4),
                  "%s: out and the scales must be 4-byte aligned", who);
    CUtensorMap tmQ, tmK, tmV;
    int rc;
    const uint32_t box_qk[2] = {64, 128}, box_v[2] = {128, 64};
    const uint64_t dq[2] = {(uint64_t)cols, (uint64_t)B * Lq}, dk[2] = {(uint64_t)cols, (uint64_t)B * Lk};
    const uint64_t dv[2] = {(uint64_t)(Lk + 15) / 16 * 16, (uint64_t)B * H * 64};
    const uint64_t stq[1] = {(uint64_t)ldq}, stk[1] = {(uint64_t)ldk}, stv[1] = {(uint64_t)ld_vt};
    if ((rc = make_tmap_16(&tmQ, CU_TENSOR_MAP_DATA_TYPE_UINT8, q8, 2, dq, stq, box_qk, 64, nullptr, 1))) return rc;
    if ((rc = make_tmap_16(&tmK, CU_TENSOR_MAP_DATA_TYPE_UINT8, k8, 2, dk, stk, box_qk, 64, nullptr, 1))) return rc;
    if ((rc = make_tmap_16(&tmV, CU_TENSOR_MAP_DATA_TYPE_UINT8, vt8, 2, dv, stv, box_v, 128, nullptr, 1))) return rc;
    AttnFp8Params p{};
    p.Lq = Lq; p.Lk = Lk; p.H = H;
    p.ldo = ldo;
    p.out = reinterpret_cast<__nv_bfloat16*>(out);
    p.sq = sq; p.sk = sk; p.sv = sv;
    p.scale_log2 = scale * 1.4426950408889634f;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    static bool attr_set[64] = {};
    const int dslot = current_device_slot();
    if (!attr_set[dslot]) {
        SUPIR_CHECK_CUDA(cudaFuncSetAttribute(attention_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AF8_SMEM));
        attr_set[dslot] = true;
    }
    const dim3 grid((Lq + AF8_BM - 1) / AF8_BM, H, B);
    attention_fp8_kernel<<<grid, AF8_THREADS, AF8_SMEM, st>>>(tmQ, tmK, tmV, p);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}
