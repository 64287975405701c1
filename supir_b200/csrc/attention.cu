// supir_b200 — K6 of SURVEY.md §2a: softmax(Q K^T / sqrt(d)) V without mask, flash-style on Hopper wgmma.
//
// Replaces F.scaled_dot_product_attention / xformers.memory_efficient_attention in CrossAttention
// (sgm/modules/attention.py:273-277, 357-359) for self-attention, 77-token cross-attention and ZeroCrossAttn
// (SUPIR/modules/SUPIR_v0.py:146), and the single-head attention of the SDXL VAE's mid block
// (sgm/modules/diffusionmodules/model.py:158-206 / MemoryEfficientAttnBlock :209-262; per tile in SUPIR/utils/tilevae.py:292-336).
//
// One kernel template serves both: a CTA owns 128 queries of one (batch, head) and DV = 64 * NVC value columns of it;
// 384 threads = three warpgroups:
//   warpgroup 0, thread 0 : TMA producer. Q (128 x D, as D / 64 chunks of 64 columns, 128B-swizzled) once; then K and V
//                           blocks of BKV keys through one ring of slots, in the order the consumers use them:
//                           K(j) chunks 0..NCH-1, V(j) chunks 0..NVC-1, K(j+1) ...
//   warpgroups 1, 2       : 64 query rows each. Per key block j:
//                             S = Q K_j^T       wgmma m64 x BKV, A and B from shared memory (both K-major)
//                             online softmax on the S fragment in registers (row max / sum across the 4 threads of a row)
//                             O += P V_j        wgmma m64 x 64 per value chunk, A = P straight from registers (the S
//                                               fragment repacked to E: accumulator and A-operand layouts coincide),
//                                               B = V in its natural [key, channel] layout (MN-major, transposed operand)
//                           and finally O / l stored as E.
// E is the 16-bit storage type (common.cuh): Bf16, or F16 for supir_attention_f16 (head_dim 64 only), whose P is packed with
// cvt.rn.f16x2.f32.
// Head dim 64 (multi-head): NCH = NVC = 1, BKV = 128. The VAE's single head of 512 channels: Q stays resident (128 KB),
// BKV = 64 keys per block (S: 32 registers per thread next to 128 of O), the 512 value columns split over two CTAs
// (grid.y), which both compute Q K^T.
#include "common.cuh"
#include "supir_b200.h"
#include "wgmma.cuh"

#include <cstdlib>

namespace supir {

static constexpr int ATT_BM = 128;   // queries per CTA (64 per consumer warpgroup)
static constexpr int ATT_THREADS = 384;

struct AttnParams {
    int Lq, Lk;
    int nsplit;            // CTAs sharing one head's value columns (grid.y = heads * nsplit)
    int head_cols;         // columns of one head in q / k / v / out
    long long ldo;
    void* out;             // E
    float scale_log2;
};

// fp32 pair -> bf16x2 with INTEGER arithmetic: round half up on the magnitude (+0x8000, p >= 0) and take the two high halves
// with one byte permute, on the ALU pipe instead of the conversion unit. Differs from round-to-nearest-even only on exact ties.
__device__ __forceinline__ uint32_t pack_bf16x2_alu(float lo, float hi) {
    return __byte_perm(__float_as_uint(lo) + 0x8000u, __float_as_uint(hi) + 0x8000u, 0x7632);
}

template <int NCH, int NVC, int BKV>
struct AttnSmem {
    static constexpr int Q_CHUNK = ATT_BM * 64 * 2;                 // 16 KB: 128 rows x 64 bf16
    static constexpr int SLOT = BKV * 64 * 2;                        // one K or V chunk: BKV rows x 64 bf16
    static constexpr int SLOTS = (NCH > NVC ? NCH : NVC) + 2 > 6 ? (NCH > NVC ? NCH : NVC) + 2 : 6;
    static constexpr int OFF_RING = NCH * Q_CHUNK;
    static constexpr int OFF_BAR = OFF_RING + SLOTS * SLOT;
    static constexpr int TOTAL = OFF_BAR + 256 + 1024;
};

template <int BKV, class E>
__device__ __forceinline__ void wgmma_qk(float (&s)[BKV / 2], uint64_t da, uint64_t db, int scale_d) {
    if constexpr (BKV == 128) wgmma_ss_n128<E>(s, da, db, scale_d);
    else wgmma_ss_n64<E>(s, da, db, scale_d);
}

// NCH = 64-column chunks of the head dim (Q K^T depth), NVC = 64-column value chunks per CTA, BKV = keys per block,
// EMU = exponential pairs of every 4 evaluated by ex2_emulated, ICVT = probability pairs of every 4 packed on the ALU pipe
// (bf16 only: the integer packing takes the high half of the fp32 bits, which is a bf16 value and not an fp16 one)
template <class E, int NCH, int NVC, int BKV, int EMU, int ICVT>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
    static_assert(ICVT == 0 || !E::kF16, "ALU packing of P produces bf16 values");
    using SM = AttnSmem<NCH, NVC, BKV>;
    constexpr int SLOTS = SM::SLOTS;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* ring = smem + SM::OFF_RING;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SM::OFF_BAR);
    uint64_t* q_full = bars;                        // 1
    uint64_t* slot_full = bars + 1;                 // [SLOTS]
    uint64_t* slot_empty = slot_full + SLOTS;       // [SLOTS]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * ATT_BM, head = blockIdx.y / p.nsplit, split = blockIdx.y % p.nsplit, batch = blockIdx.z;
    const int nblk = (p.Lk + BKV - 1) / BKV;
    const int qk_col = head * p.head_cols;                       // first Q / K column of this head
    const int v_col = head * p.head_cols + split * NVC * 64;    // first value (and output) column of this CTA

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        mbar_init(q_full, 1);
        for (int s = 0; s < SLOTS; ++s) { mbar_init(&slot_full[s], 1); mbar_init(&slot_empty[s], 8); }   // 8 consumer warps
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            mbar_expect_tx(q_full, NCH * SM::Q_CHUNK);
            for (int c = 0; c < NCH; ++c) tma_load_2d(sQ + c * SM::Q_CHUNK, &tmQ, q_full, qk_col + c * 64, batch * p.Lq + q0);
            int slot = 0;
            uint32_t phase = 0;
            auto push = [&](const CUtensorMap* tm, int col, int row) {
                mbar_wait(&slot_empty[slot], phase ^ 1);
                mbar_expect_tx(&slot_full[slot], SM::SLOT);
                tma_load_2d(ring + slot * SM::SLOT, tm, &slot_full[slot], col, row);
                if (++slot == SLOTS) { slot = 0; phase ^= 1; }
            };
            for (int j = 0; j < nblk; ++j) {
                const int row = batch * p.Lk + j * BKV;
                for (int c = 0; c < NCH; ++c) push(&tmK, qk_col + c * 64, row);
                for (int d = 0; d < NVC; ++d) push(&tmV, v_col + d * 64, row);
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int wg = (warp - 4) >> 2;                              // query rows [64 wg, 64 wg + 64) of the CTA
        const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // fragment rows r_lo and r_lo + 8
        const int cq = 2 * (lane & 3);
        int slot = 0;
        uint32_t phase = 0;
        float o[NVC][32];
#pragma unroll
        for (int d = 0; d < NVC; ++d)
#pragma unroll
            for (int i = 0; i < 32; ++i) o[d][i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        mbar_wait(q_full, 0);
        for (int j = 0; j < nblk; ++j) {
            // ---- S = Q K_j^T ----
            float s[BKV / 2];
            const int first_slot = slot;
            {
                int sl = slot;
                uint32_t ph = phase;
                for (int c = 0; c < NCH; ++c) { mbar_wait(&slot_full[sl], ph); if (++sl == SLOTS) { sl = 0; ph ^= 1; } }
            }
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const uint32_t qa = smem_u32(sQ + c * SM::Q_CHUNK + wg * 64 * 128);
                const uint32_t ka = smem_u32(ring + slot * SM::SLOT);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wgmma_qk<BKV, E>(s, wgmma_desc_sw128(qa + 32 * kk), wgmma_desc_sw128(ka + 32 * kk), (c | kk) != 0);
                if (++slot == SLOTS) { slot = 0; phase ^= 1; }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_operands(s);
            __syncwarp();
            if (lane == 0)
                for (int c = 0, sl = first_slot; c < NCH; ++c, sl = (sl + 1 == SLOTS ? 0 : sl + 1)) mbar_arrive(&slot_empty[sl]);

            // ---- online softmax on the fragment: element 4 t + 2 h + e = row r_lo + 8 h, key 8 t + cq + e ----
            const int kv_valid = min(BKV, p.Lk - j * BKV);
            if (kv_valid < BKV) {
#pragma unroll
                for (int t = 0; t < BKV / 8; ++t)
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (8 * t + cq + (e & 1) >= kv_valid) s[4 * t + e] = -INFINITY;
            }
            float alpha[2], negm[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float mx = -INFINITY;
#pragma unroll
                for (int t = 0; t < BKV / 8; ++t) mx = fmaxf(mx, fmaxf(s[4 * t + 2 * h], s[4 * t + 2 * h + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[h], mx * p.scale_log2);     // every block holds >= 1 valid key: finite
                alpha[h] = ex2_approx(m_run[h] - m_new);                    // 0 on the first block
                m_run[h] = m_new;
                negm[h] = -m_new;
                l_run[h] *= alpha[h];
            }
#pragma unroll
            for (int d = 0; d < NVC; ++d)
#pragma unroll
                for (int i = 0; i < 32; ++i) o[d][i] *= alpha[(i >> 1) & 1];
            uint32_t pa[BKV / 16][4];                                       // P as m64k16 A fragments, one per 16 keys
#pragma unroll
            for (int t = 0; t < BKV / 8; ++t) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float x0 = fmaf(s[4 * t + 2 * h], p.scale_log2, negm[h]);
                    const float x1 = fmaf(s[4 * t + 2 * h + 1], p.scale_log2, negm[h]);
                    const int q = (2 * t + h) & 3;                          // pair index inside a group of 4
                    const bool emulate = (EMU == 4) || (EMU == 3 && q != 1) || (EMU == 2 && (q & 1)) || (EMU == 1 && q == 3);
                    const float e0 = emulate ? ex2_emulated(x0) : ex2_approx(x0);
                    const float e1 = emulate ? ex2_emulated(x1) : ex2_approx(x1);
                    l_run[h] += e0 + e1;
                    const bool alu_pack = (ICVT == 4) || (ICVT == 2 && !(q & 1)) || (ICVT == 1 && q == 0) || (ICVT == 3 && q != 2);
                    // A fragment of k-step t/2: regs {0, 1} = keys [0, 8) of the step for rows r, r + 8; {2, 3} = keys [8, 16)
                    pa[t >> 1][(t & 1) * 2 + h] = alu_pack ? pack_bf16x2_alu(e0, e1) : E::pack2(e0, e1);
                }
            }

            // ---- O += P V_j ----
            const int v_first = slot;
            {
                int sl = slot;
                uint32_t ph = phase;
                for (int d = 0; d < NVC; ++d) { mbar_wait(&slot_full[sl], ph); if (++sl == SLOTS) { sl = 0; ph ^= 1; } }
            }
            wgmma_fence();
#pragma unroll
            for (int d = 0; d < NVC; ++d) {
                const uint32_t va = smem_u32(ring + slot * SM::SLOT);
#pragma unroll
                for (int kk = 0; kk < BKV / 16; ++kk)      // 16 keys = 16 rows of 128 B = two 8-row swizzle atoms
                    wgmma_rs_n64_tb<E>(o[d], pa[kk], wgmma_desc_sw128(va + kk * 2048), 1);
                if (++slot == SLOTS) { slot = 0; phase ^= 1; }
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int d = 0; d < NVC; ++d) wgmma_fence_operands(o[d]);
            __syncwarp();
            if (lane == 0)
                for (int d = 0, sl = v_first; d < NVC; ++d, sl = (sl + 1 == SLOTS ? 0 : sl + 1)) mbar_arrive(&slot_empty[sl]);
        }

        // ---- O / l -> E ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float l = l_run[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = 1.f / l;
            const int qrow = q0 + r_lo + 8 * h;
            if (qrow < p.Lq) {
                typename E::T* dst = reinterpret_cast<typename E::T*>(p.out) + ((long long)batch * p.Lq + qrow) * p.ldo + v_col + cq;
#pragma unroll
                for (int d = 0; d < NVC; ++d)
#pragma unroll
                    for (int t = 0; t < 8; ++t)
                        *reinterpret_cast<uint32_t*>(dst + d * 64 + 8 * t) =
                            E::pack2(o[d][4 * t + 2 * h] * inv, o[d][4 * t + 2 * h + 1] * inv);
            }
        }
    }
}

static int g_att_emu = -1;            // emulated exponent pairs per 4: -1 = environment / default
static int g_att_icvt = -1;           // pairs of every 4 packed to bf16 on the ALU pipe: -1 = environment / default

static int attention_int_pack() {
    if (g_att_icvt < 0) {
        const char* e = getenv("SUPIR_B200_ATTN_ALU_PACK");
        g_att_icvt = e ? atoi(e) : 0;
        if (g_att_icvt < 0 || g_att_icvt > 4) g_att_icvt = 0;
    }
    return g_att_icvt;
}

static int attention_emu() {
    if (g_att_emu < 0) {
        const char* e = getenv("SUPIR_B200_ATTN_EMU");
        g_att_emu = e ? atoi(e) : 0;
        if (g_att_emu < 0 || g_att_emu > 4) g_att_emu = 0;
    }
    return g_att_emu;
}

template <class E, int NCH, int NVC, int BKV, int EMU, int ICVT>
static int launch_attention(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const AttnParams& p,
                            int heads, int B, cudaStream_t st) {
    using SM = AttnSmem<NCH, NVC, BKV>;
    static bool attr_set[64] = {};
    const int dslot = current_device_slot();
    if (!attr_set[dslot]) {
        SUPIR_CHECK_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel<E, NCH, NVC, BKV, EMU, ICVT>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, SM::TOTAL));
        attr_set[dslot] = true;
    }
    const dim3 grid((p.Lq + ATT_BM - 1) / ATT_BM, heads * p.nsplit, B);
    attention_wgmma_kernel<E, NCH, NVC, BKV, EMU, ICVT><<<grid, ATT_THREADS, SM::TOTAL, st>>>(tmQ, tmK, tmV, p);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

static int make_attention_maps(CUtensorMapDataType dt, CUtensorMap* tmQ, CUtensorMap* tmK, CUtensorMap* tmV, const void* q, long long ldq, const void* k,
                               long long ldk, const void* v, long long ldv, uint64_t cols, uint64_t rows_q, uint64_t rows_kv,
                               uint32_t bkv) {
    int rc;
    const uint32_t box_q[2] = {64, ATT_BM}, box_kv[2] = {64, bkv};
    const uint64_t dq[2] = {cols, rows_q}, dkv[2] = {cols, rows_kv};
    const uint64_t sq[1] = {(uint64_t)ldq}, sk[1] = {(uint64_t)ldk}, sv[1] = {(uint64_t)ldv};
    if ((rc = make_tmap_16(tmQ, dt, q, 2, dq, sq, box_q))) return rc;
    if ((rc = make_tmap_16(tmK, dt, k, 2, dkv, sk, box_kv))) return rc;
    return make_tmap_16(tmV, dt, v, 2, dkv, sv, box_kv);
}

}  // namespace supir

using namespace supir;

extern "C" int supir_set_attention_alu_pack(int pairs_of_4) {
    g_att_icvt = pairs_of_4 < 0 ? -1 : (pairs_of_4 > 4 ? 4 : pairs_of_4);
    return SUPIR_OK;
}

extern "C" int supir_set_attention_exp_emulation(int pairs_of_4) {
    g_att_emu = pairs_of_4 < 0 ? -1 : (pairs_of_4 > 4 ? 4 : pairs_of_4);
    return SUPIR_OK;
}

// head_dim-64 multi-head attention: argument checks and tensor maps shared by the bf16 and fp16 entry points
static int attention_h64_setup(const char* who, CUtensorMapDataType dt, CUtensorMap* tmQ, CUtensorMap* tmK, CUtensorMap* tmV,
                               AttnParams* p, const void* q, long long ldq, const void* k, long long ldk, const void* v,
                               long long ldv, void* out, long long ldo, int B, int H, int Lq, int Lk, int head_dim, float scale) {
    SUPIR_REQUIRE(q && k && v && out, "%s: null pointer", who);
    SUPIR_REQUIRE(head_dim == 64, "%s: head_dim %d unsupported (64 only; the VAE's single wide head is supir_attention_1head_bf16)", who, head_dim);
    SUPIR_REQUIRE(B > 0 && H > 0 && Lq > 0 && Lk > 0, "%s: bad shape", who);
    SUPIR_REQUIRE(scale > 0.f, "%s: scale must be positive", who);
    SUPIR_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "%s: leading dims must be multiples of 8", who);
    const long long cols = (long long)H * 64;
    SUPIR_REQUIRE(ldq >= cols && ldk >= cols && ldv >= cols && ldo >= cols, "%s: leading dims must be >= H * 64 = %lld", who, cols);
    // the final store writes two outputs as one 32-bit word
    SUPIR_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "%s: out must be 4-byte aligned", who);
    int rc = make_attention_maps(dt, tmQ, tmK, tmV, q, ldq, k, ldk, v, ldv, (uint64_t)H * 64, (uint64_t)B * Lq, (uint64_t)B * Lk, 128);
    if (rc) return rc;
    *p = AttnParams{};
    p->Lq = Lq; p->Lk = Lk;
    p->nsplit = 1;
    p->head_cols = 64;
    p->ldo = ldo;
    p->out = out;
    p->scale_log2 = scale * 1.4426950408889634f;
    return SUPIR_OK;
}

extern "C" int supir_attention_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                    long long ldv, void* out, long long ldo, int B, int H, int Lq, int Lk, int head_dim,
                                    float scale, void* stream) {
    CUtensorMap tmQ, tmK, tmV;
    AttnParams p;
    int rc = attention_h64_setup("supir_attention_bf16", Bf16::kTma, &tmQ, &tmK, &tmV, &p, q, ldq, k, ldk, v, ldv, out, ldo, B, H,
                                 Lq, Lk, head_dim, scale);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (attention_emu() >= 2) return launch_attention<Bf16, 1, 1, 128, 2, 0>(tmQ, tmK, tmV, p, H, B, st);
    switch (attention_int_pack()) {
        case 0: return launch_attention<Bf16, 1, 1, 128, 0, 0>(tmQ, tmK, tmV, p, H, B, st);
        case 1: case 2: return launch_attention<Bf16, 1, 1, 128, 0, 2>(tmQ, tmK, tmV, p, H, B, st);
        case 3: return launch_attention<Bf16, 1, 1, 128, 0, 3>(tmQ, tmK, tmV, p, H, B, st);
        default: return launch_attention<Bf16, 1, 1, 128, 0, 4>(tmQ, tmK, tmV, p, H, B, st);
    }
}

// fp16: the ALU-packing knob (supir_set_attention_alu_pack) has no effect here; P always goes through cvt.rn.f16x2.f32
extern "C" int supir_attention_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                   long long ldv, void* out, long long ldo, int B, int H, int Lq, int Lk, int head_dim,
                                   float scale, void* stream) {
    CUtensorMap tmQ, tmK, tmV;
    AttnParams p;
    int rc = attention_h64_setup("supir_attention_f16", F16::kTma, &tmQ, &tmK, &tmV, &p, q, ldq, k, ldk, v, ldv, out, ldo, B, H,
                                 Lq, Lk, head_dim, scale);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (attention_emu() >= 2) return launch_attention<F16, 1, 1, 128, 2, 0>(tmQ, tmK, tmV, p, H, B, st);
    return launch_attention<F16, 1, 1, 128, 0, 0>(tmQ, tmK, tmV, p, H, B, st);
}

extern "C" int supir_attention_1head_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                          long long ldv, void* out, long long ldo, int B, int L, int head_dim, float scale,
                                          void* stream) {
    SUPIR_REQUIRE(q && k && v && out, "supir_attention_1head_bf16: null pointer");
    SUPIR_REQUIRE(B > 0 && L > 0 && scale > 0.f, "supir_attention_1head_bf16: bad shape");
    SUPIR_REQUIRE(head_dim == 512 || head_dim == 256 || head_dim == 128, "supir_attention_1head_bf16: head_dim %d not in {128, 256, 512}", head_dim);
    SUPIR_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && ldq >= head_dim && ldk >= head_dim && ldv >= head_dim && ldo >= head_dim,
                  "supir_attention_1head_bf16: leading dims must be multiples of 8 and >= head_dim");
    SUPIR_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "supir_attention_1head_bf16: out must be 4-byte aligned");
    CUtensorMap tmQ, tmK, tmV;
    int rc = make_attention_maps(Bf16::kTma, &tmQ, &tmK, &tmV, q, ldq, k, ldk, v, ldv, (uint64_t)head_dim, (uint64_t)B * L, (uint64_t)B * L, 64);
    if (rc) return rc;
    AttnParams p{};
    p.Lq = L; p.Lk = L;
    p.head_cols = head_dim;
    p.nsplit = head_dim == 512 ? 2 : 1;          // at most 256 value columns (128 fp32 registers of O per thread) per CTA
    p.ldo = ldo;
    p.out = out;
    p.scale_log2 = scale * 1.4426950408889634f;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int emu = attention_emu();
    if (head_dim == 512) {
        if (emu == 2) return launch_attention<Bf16, 8, 4, 64, 2, 0>(tmQ, tmK, tmV, p, 1, B, st);
        if (emu == 4) return launch_attention<Bf16, 8, 4, 64, 4, 0>(tmQ, tmK, tmV, p, 1, B, st);
        return launch_attention<Bf16, 8, 4, 64, 0, 0>(tmQ, tmK, tmV, p, 1, B, st);
    }
    if (head_dim == 256) return launch_attention<Bf16, 4, 4, 64, 0, 0>(tmQ, tmK, tmV, p, 1, B, st);
    return launch_attention<Bf16, 2, 2, 64, 0, 0>(tmQ, tmK, tmV, p, 1, B, st);
}
