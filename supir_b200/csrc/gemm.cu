// supir_b200 — K2/K3/K4 of SURVEY.md §2a: Linear, conv1x1 and conv3x3 (implicit GEMM) on Hopper wgmma.
//
//   out[m, n] = epilogue( sum_k A[m, k] * W[n, k] )          E x E -> fp32 (registers) -> E/fp32
//
// E is the 16-bit storage type (common.cuh): Bf16 (supir_gemm_bf16 ...) or F16 (the _f16 twins). Every rounding point of
// the epilogue rounds to E. E4m3 (supir_gemm_fp8, supir_conv3x3_fp8) is Bf16 storage with e4m3 operands: A and W hold e4m3
// codes, and the epilogue first multiplies the accumulator by a_scale[m] * w_scale[n] (per-row scales of both operands; in conv
// mode a_scale is per image, a_scale[image of m]).
//
// Replaces, on the sampling path of the reference: nn.Linear (sgm/modules/attention.py:213-218,87,106,587,611),
// nn.Conv2d 1x1 (openaimodel.py:317, SUPIR_v0.py:48,87, model.py:124-126,164-175) and nn.Conv2d 3x3 stride 1 pad 1
// (openaimodel.py:263,300-307; SUPIR_v0.py:79,82-83; model.py:108-117 ...).
//
// Design (one persistent CTA per SM, 384 threads = three warpgroups, warp-specialised):
//   warpgroup 0, thread 0 : TMA producer.  A tile = 128 rows x 64 k (bf16; 128 k of e4m3: 128B-swizzled), W tile = BN rows x 64 k.
//                   GEMM mode: A is a 2-D tensor map over [M, K].
//                   CONV mode: A is a 4-D tensor map over the NHWC activation [B, H, W, C]; the tile's 128 rows are a
//                   TH x TW pixel patch and the k-loop runs over (tap, BK-channel chunk); the tap shift is applied to the
//                   TMA coordinates, and TMA's out-of-bounds zero fill IS the conv padding (no im2col buffer).
//   warpgroups 1, 2       : wgmma consumers (m64nBNk16, fp32 accumulators in registers, one wgmma group kept in flight).
//                   BN in {160, 256}, cooperative: rows [0, 64) and [64, 128) of every tile. BN in {64, 128}, ping-pong: each
//                   warpgroup owns alternate whole tiles, and one's epilogue runs under the other's mainloop.
//                   Then the epilogue from the accumulator fragment:
//                   +bias, +per-batch vector (timestep embedding), folded LayerNorm, SiLU / GEGLU, bf16 round, +residual.
//                   16-bit outputs go through a shared-memory staging buffer and TMA stores (the residual arrives there
//                   by TMA during the mainloop); fp32 and unaligned outputs are stored directly. The producer keeps
//                   filling the shared-memory ring for the next tile meanwhile.
// Pipeline: smem full/empty mbarrier ring (TMA <-> wgmma).
#include "common.cuh"
#include "supir_b200.h"
#include "wgmma.cuh"

#include <mutex>

namespace supir {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int GEMM_THREADS = 384;   // warpgroup 0: TMA; warpgroups 1, 2: wgmma + epilogue (64 rows each)

struct GemmKernelParams {
    int M, N, K;          // N = accumulator columns (before GEGLU halving)
    int num_m_tiles, num_n_tiles, num_kb;
    int m_fastest;        // tile order: 1 = consecutive tiles share the W tile, 0 = they share the A tile
    // conv mode
    int conv;             // 0 gemm, 1 conv3x3
    int H, W, Cin, TH, TW, tiles_x, tiles_y, kchunks;   // H, W: OUTPUT grid of the convolution
    // conv geometry (supir_conv_geometry): taps kh x ntaps_x, input pixel of tap (ky, kx) for output (y, x) =
    // (y * stride + ky + off_y, x * stride + kx + off_x); out-of-image taps read TMA's zero fill
    int ntaps_x, stride, off_y, off_x;
    // where output pixel (y, x) lands in the output tensor [nimg, out_H, out_W, ldc]: (y * out_sy + out_oy, x * out_sx + out_ox)
    int out_sy, out_sx, out_oy, out_ox, out_H, out_W;
    // epilogue
    const float* bias;
    const float* rowvec;
    int rows_per_batch;
    int rowvec_ld;
    const void* residual;     // E [M, ldr]
    long long ldr;
    int act;
    void* out;
    long long ldc;
    int out_f32;
    int n_out;            // valid output columns (N or N/2 for GEGLU)
    int nimg;             // conv mode: number of images
    const float2* ln_stats;  // per-row (rstd, mean * rstd) of A: LayerNorm folded into the epilogue (see supir_epilogue), or null
    const float* ln_colsum;  // [N] row sums of the (gamma-scaled) weight matrix
    int staged;           // 1: the epilogue goes through shared memory and TMA (tmO / tmR); 0: direct global stores
    const float* a_scale;    // E4m3 only: [M] dequantization scale of each row of A (conv mode: [nimg], one per image)
    const float* w_scale;    // E4m3 only: [N] dequantization scale of each row of W (accumulator column)
};

// tile widths 64 and 128 run the ping-pong schedule (each consumer warpgroup owns whole 128 x BN tiles, BN accumulators per
// thread); 160 and 256 run the cooperative one (both warpgroups on one tile, BN / 2 accumulators per thread)
__host__ __device__ constexpr bool gemm_pingpong(int bn) { return bn <= 128; }

// Shared memory: the operand ring, then the staged epilogue's buffer (one per consumer warpgroup: the 128 x BN tile it owns
// under ping-pong, its 64 x BN half under the cooperative schedule), then the barriers. The ring takes as many stages (<= 8)
// as fit next to the staging buffers in the 227 KB opt-in limit: 8 / 5 / 5 / 3 stages at BN = 64 / 128 / 160 / 256.
template <int BN>
struct GemmSmem {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int FRAG_BYTES = 64 * BN * 2;                                 // one 64-row fragment of 16-bit outputs
    static constexpr int EPI_BYTES = 2 * (gemm_pingpong(BN) ? 2 : 1) * FRAG_BYTES;  // both consumer warpgroups
    static constexpr int BAR_BYTES = 256;
    static constexpr int FIT = (227 * 1024 - EPI_BYTES - BAR_BYTES - 1024) / STAGE_BYTES;
    static constexpr int STAGES = FIT > 8 ? 8 : FIT;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + EPI_BYTES + BAR_BYTES + 1024;  // +1024 alignment slack
    static_assert(STAGES >= 3 && TOTAL <= 227 * 1024, "GEMM shared memory does not fit");
};

// Staged epilogue layout: a 64-row fragment is stored as 32-column slabs of 64 rows x 64 bytes, each slab in the 64-byte
// swizzle of a SWIZZLE_64B tensor map (16-byte chunk index XOR (row / 2) % 4), so the accumulator fragment's column-pair
// writes are free of bank conflicts and one TMA box moves one slab. Byte offset of output columns (c, c + 1) of row r:
__device__ __forceinline__ uint32_t stage_off(int r, int c) {
    return (c >> 5) * 4096 + r * 64 + ((((c >> 3) & 3) ^ ((r >> 1) & 3)) << 4) + (c & 7) * 2;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v));
}
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

template <int BN, class E>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
    if constexpr (BN == 256) wgmma_ss_n256<E>(d, da, db, scale_d);
    else if constexpr (BN == 160) wgmma_ss_n160<E>(d, da, db, scale_d);
    else if constexpr (BN == 128) wgmma_ss_n128<E>(d, da, db, scale_d);
    else wgmma_ss_n64<E>(d, da, db, scale_d);
}

// two adjacent output columns (n, n + 1) of one row; `n1ok`: column n + 1 exists
template <class E>
__device__ __forceinline__ void store_pair(const GemmKernelParams& p, long long grow, int n, float v0, float v1, bool n1ok) {
    if (p.out_f32) {
        float* dst = reinterpret_cast<float*>(p.out) + grow * p.ldc + n;
        if (n1ok && ((reinterpret_cast<uintptr_t>(dst) & 7) == 0)) { *reinterpret_cast<float2*>(dst) = make_float2(v0, v1); }
        else { dst[0] = v0; if (n1ok) dst[1] = v1; }
    } else {
        typename E::T* dst = reinterpret_cast<typename E::T*>(p.out) + grow * p.ldc + n;
        if (n1ok && ((reinterpret_cast<uintptr_t>(dst) & 3) == 0)) { *reinterpret_cast<uint32_t*>(dst) = E::pack2(v0, v1); }
        else { dst[0] = E::from_f(v0); if (n1ok) dst[1] = E::from_f(v1); }
    }
}
// residual pair (n, n + 1) as the packed bits of two E values; a missing column n + 1 reads as 0
template <class E>
__device__ __forceinline__ uint32_t load_res_bits(const GemmKernelParams& p, long long grow, int n, bool n1ok) {
    const typename E::T* src = reinterpret_cast<const typename E::T*>(p.residual) + grow * p.ldr + n;
    if (n1ok && ((reinterpret_cast<uintptr_t>(src) & 3) == 0)) return __ldg(reinterpret_cast<const unsigned int*>(src));
    const uint32_t lo = E::bits(src[0]);
    return n1ok ? lo | (E::bits(src[1]) << 16) : lo;
}

// m-tile and n-tile of persistent tile index `tile` (tile order: m_fastest)
__device__ __forceinline__ void tile_coords(const GemmKernelParams& p, int tile, int& mt, int& nt) {
    mt = p.m_fastest ? tile % p.num_m_tiles : tile / p.num_n_tiles;
    nt = p.m_fastest ? tile / p.num_m_tiles : tile % p.num_n_tiles;
}

// conv mode: image b and output pixel (y, x) of row r of m-tile mt (its rows are a TH x TW pixel patch, row-major)
__device__ __forceinline__ void conv_pixel(const GemmKernelParams& p, int mt, int r, int& b, int& y, int& x) {
    const int per_img = p.tiles_x * p.tiles_y;
    b = mt / per_img;
    const int t = mt % per_img;
    y = (t / p.tiles_x) * p.TH + r / p.TW;
    x = (t % p.tiles_x) * p.TW + r % p.TW;
}

// output row of accumulator row `row_in_tile` of m-tile `mt`: its row index in the output / residual, its image (per-batch
// vector index) and whether it exists
struct EpiRow {
    long long grow;
    int batch;
    bool ok;
};
__device__ __forceinline__ EpiRow epi_row(const GemmKernelParams& p, int mt, int row_in_tile) {
    EpiRow r;
    if (p.conv) {
        int b, y, x;
        conv_pixel(p, mt, row_in_tile, b, y, x);
        r.ok = (y < p.H) && (x < p.W) && (b < p.nimg);
        r.grow = ((long long)b * p.out_H + (long long)y * p.out_sy + p.out_oy) * p.out_W + (long long)x * p.out_sx + p.out_ox;
        r.batch = b;
    } else {
        r.grow = (long long)mt * BM + row_in_tile;
        r.ok = r.grow < p.M;
        r.batch = p.rows_per_batch > 0 ? (int)(r.grow / p.rows_per_batch) : 0;
    }
    return r;
}

// This thread's columns of a fragment as pairs: s[j] = (src[n], src[n + 1]) for n = n0 + 8 j (n0 even), all at fixed offsets
// from one address. One 64-bit load per pair when every column is inside N (`full`) and `src` is 8-byte aligned; otherwise
// two 32-bit loads, and columns past N read as 0 (their results are never stored).
template <int NJ>
__device__ __forceinline__ void load_col_pairs(float2 (&s)[NJ], const float* src, int n0, int N, bool full) {
    if (full && (reinterpret_cast<uintptr_t>(src) & 7) == 0) {
        const float2* q = reinterpret_cast<const float2*>(src + n0);
#pragma unroll
        for (int j = 0; j < NJ; ++j) s[j] = __ldg(q + 4 * j);
    } else {
        const float* q = src + n0;
#pragma unroll
        for (int j = 0; j < NJ; ++j)
            s[j] = make_float2(n0 + 8 * j < N ? __ldg(q + 8 * j) : 0.f, n0 + 8 * j + 1 < N ? __ldg(q + 8 * j + 1) : 0.f);
    }
}

// f(j, pair j) for every column pair j < NJ of this thread: one branch-free pass that issues all of its loads before the
// first use
template <int NJ, class F>
__device__ __forceinline__ void col_pass(const float* src, int n0, int N, bool full, F&& f) {
    float2 s[NJ];
    load_col_pairs(s, src, n0, N, full);
#pragma unroll
    for (int j = 0; j < NJ; ++j) f(j, s[j]);
}

// Epilogue of one m64 accumulator fragment of tile (mt, nt): rows [row0, row0 + 64) of the tile, of which this thread holds
// rows row0 + r_lo and row0 + r_lo + 8 (h = 0, 1: v[4 j + 2 h + e]), columns 8 j + cq + e. STAGED: the residual is read
// from, and the output written to, the fragment's staging buffer at shared address `frag` (stage_off layout; the residual was
// put there by TMA), and TMA stores it afterwards; rows and columns outside the output are skipped here and clipped by the
// store. Otherwise both go straight to global memory. The arithmetic and its rounding points are the same either way.
// The epilogue works on the accumulators in place (a copy would not fit in registers beside them: the next tile's wgmma
// keeps them live, and overwrites them). Both rows share their columns, so each column operand is loaded once per fragment,
// as pairs, in one branch-free pass (col_pass) applied to both rows; the per-row terms are loaded once per row.
template <int BN, bool STAGED, class E>
__device__ __forceinline__ void epilogue_m64(const GemmKernelParams& p, float (&v)[BN / 2], int mt, int nt, int row0,
                                             int r_lo, int cq, uint32_t frag) {
    constexpr int NJ = BN / 8;
    const EpiRow row[2] = {epi_row(p, mt, row0 + r_lo), epi_row(p, mt, row0 + r_lo + 8)};
    if (!row[0].ok && !row[1].ok) return;
    const int n0 = nt * BN + cq;
    const bool full = nt * BN + BN <= p.N;                    // every column of the tile is inside N
    // Per-row terms. A row outside the output borrows the other row's (its results are never stored).
    float sa[2] = {1.f, 1.f};
    float2 st[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
    const float* rv[2] = {nullptr, nullptr};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const EpiRow rw = row[h].ok ? row[h] : row[h ^ 1];
        // E4m3: the accumulator times a_scale[row] * w_scale[column] comes first (sa * w_scale[n] below); a convolution's
        // activation scale is per image (a pixel's k-sum spans 9 input pixels: only a scale they share factors out of it)
        if constexpr (E::kFp8) sa[h] = __ldg(p.a_scale + (p.conv ? (long long)rw.batch : rw.grow));
        if (p.ln_stats) st[h] = __ldg(p.ln_stats + rw.grow);
        if (p.rowvec) rv[h] = p.rowvec + (long long)rw.batch * p.rowvec_ld;
    }
    // One pass per column operand (run-time branches: they keep the passes' loads apart)
    if (E::kFp8 && p.w_scale)
        col_pass<NJ>(p.w_scale, n0, p.N, full, [&](int j, float2 s) {
#pragma unroll
            for (int h = 0; h < 2; ++h) { v[4 * j + 2 * h] *= sa[h] * s.x; v[4 * j + 2 * h + 1] *= sa[h] * s.y; }
        });
    if (p.ln_stats)
        col_pass<NJ>(p.ln_colsum, n0, p.N, full, [&](int j, float2 s) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                v[4 * j + 2 * h] = fmaf(v[4 * j + 2 * h], st[h].x, -st[h].y * s.x);
                v[4 * j + 2 * h + 1] = fmaf(v[4 * j + 2 * h + 1], st[h].x, -st[h].y * s.y);
            }
        });
    if (p.bias)
        col_pass<NJ>(p.bias, n0, p.N, full, [&](int j, float2 s) {
#pragma unroll
            for (int h = 0; h < 2; ++h) { v[4 * j + 2 * h] += s.x; v[4 * j + 2 * h + 1] += s.y; }
        });
    if (p.rowvec) {
        // one pass when both rows are in one batch (always in conv mode: a tile is one image's patch), else one per row
        const bool one = rv[0] == rv[1];
        col_pass<NJ>(rv[0], n0, p.N, full, [&](int j, float2 s) {
            v[4 * j] += s.x; v[4 * j + 1] += s.y;
            if (one) { v[4 * j + 2] += s.x; v[4 * j + 3] += s.y; }
        });
        if (!one)
            col_pass<NJ>(rv[1], n0, p.N, full, [&](int j, float2 s) { v[4 * j + 2] += s.x; v[4 * j + 3] += s.y; });
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (!row[h].ok) continue;
        const int r = r_lo + 8 * h;
        const long long grow = row[h].grow;
        if (p.act == 2) {
            // GEGLU: accumulator columns come in groups of 32 = [16 value | 16 gate]; this thread holds value column
            // 8 b + cq (+1) of group g in block 4 g + b and its gate 16 columns later in block 4 g + b + 2
            constexpr int NG = BN / 32;
#pragma unroll
            for (int g = 0; g < NG; ++g) {
                if (nt * BN + g * 32 >= p.N) break;
#pragma unroll
                for (int b = 0; b < 2; ++b) {
                    const float xv0 = v[4 * (4 * g + b) + 2 * h], xv1 = v[4 * (4 * g + b) + 2 * h + 1];
                    const float gv0 = v[4 * (4 * g + b + 2) + 2 * h], gv1 = v[4 * (4 * g + b + 2) + 2 * h + 1];
                    float o0 = E::round(E::round(xv0) * E::round(gelu_erf_f(E::round(gv0))));
                    float o1 = E::round(E::round(xv1) * E::round(gelu_erf_f(E::round(gv1))));
                    const int c = g * 16 + b * 8 + cq;                 // output column within the tile's BN / 2
                    const int oc = (nt * BN) / 2 + c;
                    if (p.residual) {
                        const float2 rr = E::unpack2(STAGED ? ld_shared_u32(frag + stage_off(r, c)) : load_res_bits<E>(p, grow, oc, true));
                        o0 += rr.x; o1 += rr.y;
                    }
                    if constexpr (STAGED) st_shared_u32(frag + stage_off(r, c), E::pack2(o0, o1));
                    else store_pair<E>(p, grow, oc, o0, o1, true);
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int n = nt * BN + 8 * j + cq;
                if (n >= p.N) break;
                const bool n1ok = n + 1 < p.N;
                float v0 = v[4 * j + 2 * h], v1 = v[4 * j + 2 * h + 1];
                if (p.act == 1) { v0 = silu_f(E::round(v0)); v1 = silu_f(E::round(v1)); }
                if (p.residual) {
                    const float2 rr = E::unpack2(STAGED ? ld_shared_u32(frag + stage_off(r, 8 * j + cq)) : load_res_bits<E>(p, grow, n, n1ok));
                    if (!STAGED && p.out_f32) { v0 += rr.x; v1 += rr.y; }
                    else { v0 = E::round(v0) + rr.x; v1 = E::round(v1) + rr.y; }
                }
                if constexpr (STAGED) st_shared_u32(frag + stage_off(r, 8 * j + cq), E::pack2(v0, v1));
                else store_pair<E>(p, grow, n, v0, v1, n1ok);
            }
        }
    }
}

// TMA coordinates of 64-row fragment f (tile rows [64 f, 64 f + 64)) of m-tile mt: GEMM (row, -), conv (x, y, image). False
// when the fragment has no row inside the output (the tail of the last m-tile, or a conv patch half below the image).
__device__ __forceinline__ bool frag_origin(const GemmKernelParams& p, int mt, int f, int& c1, int& c2, int& c3) {
    if (p.conv) {
        conv_pixel(p, mt, 64 * f, c3, c2, c1);
        return c1 < p.W && c2 < p.H;
    }
    c1 = mt * BM + 64 * f;
    c2 = c3 = 0;
    return c1 < p.M;
}

// One thread's TMA traffic for the staging buffer at `buf` (fragments f0 .. f0 + nfrag - 1 of tile (mt, nt), one per
// FRAG_BYTES): with `bar`, load the residual slabs into it (if the epilogue has a residual: tmR is only valid then) and
// arrive on `bar` with their byte count (zero bytes completes the phase at once); without, store the output slabs and
// commit them as one bulk group.
template <int BN>
__device__ __forceinline__ void epi_tma(const GemmKernelParams& p, const CUtensorMap* tm, uint8_t* buf, int f0, int nfrag, int mt,
                                        int nt, uint64_t* bar) {
    const int bno = p.act == 2 ? BN / 2 : BN;
    uint32_t bytes = 0;
    if (bar) {
        for (int f = 0; f < nfrag && p.residual; ++f) {
            int c1, c2, c3;
            if (!frag_origin(p, mt, f0 + f, c1, c2, c3)) continue;
            for (int s = 0; s < bno / 32 && nt * bno + 32 * s < p.n_out; ++s) bytes += 4096;
        }
        mbar_expect_tx(bar, bytes);
        if (bytes == 0) return;
    }
    for (int f = 0; f < nfrag; ++f) {
        int c1, c2, c3;
        if (!frag_origin(p, mt, f0 + f, c1, c2, c3)) continue;
        for (int s = 0; s < bno / 32; ++s) {
            const int c0 = nt * bno + 32 * s;
            if (c0 >= p.n_out) break;
            uint8_t* slab = buf + f * GemmSmem<BN>::FRAG_BYTES + s * 4096;
            if (bar) {
                if (p.conv) tma_load_4d(slab, tm, bar, c0, c1, c2, c3);
                else tma_load_2d(slab, tm, bar, c0, c1);
            } else {
                if (p.conv) tma_store_4d(tm, slab, c0, c1, c2, c3);
                else tma_store_2d(tm, slab, c0, c1);
            }
        }
    }
    if (!bar) bulk_commit_group();
}

template <int BN, class E>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR, const GemmKernelParams p) {
    using S = GemmSmem<BN>;
    constexpr int STAGES = S::STAGES;
    constexpr bool PINGPONG = gemm_pingpong(BN);
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * S::A_BYTES;
    uint8_t* smem_epi = smem + STAGES * S::STAGE_BYTES;                                  // [2][EPI_BYTES / 2]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_epi + S::EPI_BYTES);          // [STAGES]
    uint64_t* empty_bar = full_bar + STAGES;                                              // [STAGES]
    uint64_t* epi_bar = empty_bar + STAGES;                                               // [2]: staging buffer ready

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.num_m_tiles * p.num_n_tiles;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (p.staged) {
            tma_prefetch_desc(&tmO);
            if (p.residual) tma_prefetch_desc(&tmR);
        }
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], PINGPONG ? 4 : 8);   // one arrive per warp of the warpgroup(s) consuming the stage
        }
        mbar_init(&epi_bar[0], 1);
        mbar_init(&epi_bar[1], 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            // ===================== TMA producer =====================
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int mt, nt;
                tile_coords(p, tile, mt, nt);
                int b = 0, y0 = 0, x0 = 0;
                if (p.conv) conv_pixel(p, mt, 0, b, y0, x0);
                const int bn0 = nt * BN;
                // conv mode walks (tap row, tap column, BK-channel chunk) with counters: no division in the per-k-block path
                int cc = 0, tx = 0, ty = 0, wcol = 0;
                const int ax0 = x0 * p.stride + p.off_x, ay0 = y0 * p.stride + p.off_y;
                for (int kb = 0; kb < p.num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], S::STAGE_BYTES);
                    uint8_t* sa = smem_a + stage * S::A_BYTES;
                    uint8_t* sb = smem_b + stage * S::B_BYTES;
                    if (p.conv) {
                        tma_load_4d(sa, &tmA, &full_bar[stage], cc * E::kBK, ax0 + tx, ay0 + ty, b);
                        tma_load_2d(sb, &tmB, &full_bar[stage], wcol + cc * E::kBK, bn0);
                        if (++cc == p.kchunks) {                       // next tap: W columns advance by Cin
                            cc = 0;
                            wcol += p.Cin;
                            if (++tx == p.ntaps_x) { tx = 0; ++ty; }
                        }
                    } else {
                        tma_load_2d(sa, &tmA, &full_bar[stage], kb * E::kBK, mt * BM);
                        tma_load_2d(sb, &tmB, &full_bar[stage], kb * E::kBK, bn0);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ===================== wgmma consumers + epilogue (warpgroups 1, 2) =====================
        // Two schedules, fixed by the tile width (gemm_pingpong):
        //   ping-pong (BN 64, 128): warpgroup wg owns the CTA's tiles wg, wg + 2, ... whole (all 128 rows: FRAGS = 2 m64
        //     fragments). Their mainloops take turns on the tensor cores through named barriers 1 and 2 (warpgroup wg waits
        //     on 1 + wg before its mainloop; the other arrives on it after finishing its own), so one warpgroup's epilogue
        //     runs under the other's mainloop. A warpgroup's ring position skips the other's k-blocks. The handoff also keeps
        //     each warpgroup within one ring pass of the producer, which makes the parity waits on the full barriers
        //     unambiguous.
        //   cooperative (BN 160, 256): both warpgroups work on every tile, warpgroup wg on rows [64 wg, 64 wg + 64) (FRAGS =
        //     1, fragment wg), and both walk the whole ring in step.
        // Staged epilogue: warpgroup wg owns staging buffer wg; its first thread (the leader) issues the buffer's TMA traffic.
        // Early in each tile's mainloop (after the first k-block's wgmma is issued, so the wait overlaps the tensor cores) the
        // leader waits until the previous tile's stores have read the buffer, then loads this tile's residual into it and
        // arrives on epi_bar[wg]; the epilogue waits on that barrier, writes its results over the residual, and the leader
        // stores them. The operand producer never waits on the staging buffer.
        constexpr int FRAGS = PINGPONG ? 2 : 1;
        const int wg = (warp - 4) >> 2;
        const int frag0 = PINGPONG ? 0 : wg;                  // this warpgroup's first m64 fragment of a tile
        const int r_w = (warp & 3) * 16 + (lane >> 2);        // this thread's accumulator rows r_w and r_w + 8 of an m64 fragment
        const int cq = 2 * (lane & 3);                        // first of the two columns this thread holds per 8-column block
        uint8_t* ebuf = smem_epi + wg * (S::EPI_BYTES / 2);
        const bool leader = (threadIdx.x & 127) == 0;
        uint32_t epi_phase = 0;
        const int prefetch_kb = p.num_kb > 1 ? 1 : 0;
        float acc[FRAGS][BN / 2];
        int it = wg * p.num_kb;                               // ping-pong: ring position of this warpgroup's next k-block
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x + (PINGPONG ? wg : 0) * gridDim.x; tile < num_tiles; tile += (PINGPONG ? 2 : 1) * gridDim.x) {
            int mt, nt;
            tile_coords(p, tile, mt, nt);
            if constexpr (PINGPONG) {
                if (tile != (int)blockIdx.x) named_bar_sync(1 + wg, 256);
                stage = it % STAGES;
                phase = (it / STAGES) & 1;
            }
            int prev = -1;
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem_a + stage * S::A_BYTES + frag0 * 64 * 128);
                const uint32_t b_addr = smem_u32(smem_b + stage * S::B_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {                 // 32 bytes (16 k-elements, 32 for e4m3) inside the 128B swizzle row
                    const uint64_t db = wgmma_desc_sw128(b_addr + 32 * k);
#pragma unroll
                    for (int f = 0; f < FRAGS; ++f)
                        wgmma_tile<BN, E>(acc[f], wgmma_desc_sw128(a_addr + f * 64 * 128 + 32 * k), db, (kb | k) != 0);
                }
                wgmma_commit();
                if (kb == prefetch_kb && p.staged) {
                    if (leader) {
                        bulk_wait_group_read<0>();
                        epi_tma<BN>(p, &tmR, ebuf, frag0, FRAGS, mt, nt, &epi_bar[wg]);
                    }
                    __syncwarp();                            // wgmma.wait_group below is warp-aligned
                }
                wgmma_wait<1>();                             // the previous k-block's group has retired: its slot is free
                if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int f = 0; f < FRAGS; ++f) wgmma_fence_operands(acc[f]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            if constexpr (PINGPONG) {
                if (tile + (int)gridDim.x < num_tiles) named_bar_arrive(1 + (wg ^ 1), 256);   // the other warpgroup's turn
                it += 2 * p.num_kb;
            }
            if (p.staged) {
                mbar_wait(&epi_bar[wg], epi_phase);
                epi_phase ^= 1;
#pragma unroll
                for (int f = 0; f < FRAGS; ++f)
                    epilogue_m64<BN, true, E>(p, acc[f], mt, nt, 64 * (frag0 + f), r_w, cq, smem_u32(ebuf + f * S::FRAG_BYTES));
                fence_proxy_async_smem();
                __syncwarp();
                named_bar_sync(3 + wg, 128);
                if (leader) epi_tma<BN>(p, &tmO, ebuf, frag0, FRAGS, mt, nt, nullptr);
                __syncwarp();
            } else {
#pragma unroll
                for (int f = 0; f < FRAGS; ++f) epilogue_m64<BN, false, E>(p, acc[f], mt, nt, 64 * (frag0 + f), r_w, cq, 0);
            }
        }
        if (p.staged && leader) bulk_wait_group_read<0>();   // the last stores have read the buffer before the CTA exits
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
    static PFN_tmapEncodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_tmapEncodeTiled>(f);
    });
    return fn;
}

// Tensor map of 16-bit elements (bf16 or fp16: `dt`), or of `elem_bytes`-byte ones (e4m3 GEMM operands as UINT8); dims /
// strides innermost first, strides in ELEMENTS for dims 1..rank-1. `swizzle` in bytes: 128 for GEMM / attention operands, 64 for the staged epilogue's slabs. `elem_strides`
// (null: all 1) are traversal strides: the box spans box[i] tensor elements of dimension i and delivers every
// elem_strides[i]-th of them, densely packed (a stride-2 convolution's input patch).
int make_tmap_16(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_elems, const uint32_t* box, int swizzle, const uint32_t* elem_strides, int elem_bytes) {
    PFN_tmapEncodeTiled fn = get_encode_fn();
    if (!fn) return set_error(SUPIR_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = elem_strides ? elem_strides[i] : 1;
    }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_elems[i] * elem_bytes;
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
        return set_error(SUPIR_ERR_INVALID, "TMA base address %p is not 16-byte aligned", base);
    for (int i = 0; i + 1 < rank; ++i)
        if (gstr[i] % 16 != 0) return set_error(SUPIR_ERR_INVALID, "TMA stride %d (%llu B) not a multiple of 16", i,
                                                 (unsigned long long)gstr[i]);
    const CUtensorMapSwizzle sw = swizzle == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : swizzle == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                  : swizzle == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = fn(m, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error(SUPIR_ERR_CUDA, "cuTensorMapEncodeTiled%s failed with CUresult %d", elem_strides ? " (strided)" : "",
                         (int)r);
    return SUPIR_OK;
}

template <int BN, class E>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const CUtensorMap& tmR,
                       GemmKernelParams p, cudaStream_t st) {
    using S = GemmSmem<BN>;
    static bool attr_set[64] = {};
    const int dslot = current_device_slot();
    if (!attr_set[dslot]) {
        SUPIR_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
        attr_set[dslot] = true;
    }
    p.num_n_tiles = (p.N + BN - 1) / BN;
    {
        // tile order that minimises HBM traffic under a simple L2 model (50 MB of L2 on H100): the tiles in flight together
        // (one round: one per SM, two under ping-pong) either share a W tile (m-fastest; A is re-streamed once per n-tile
        // unless it fits L2) or share an A tile (n-fastest; W is re-streamed once per round of m-tiles unless it fits L2)
        const double l2 = 50e6;
        const double a_bytes = (double)E::kOpBytes * p.M * (p.conv ? p.Cin : p.K), w_bytes = (double)E::kOpBytes * p.N * p.K;
        const double in_flight = (double)device_sm_count() * (gemm_pingpong(BN) ? 2 : 1);
        const double rounds_m = (double)p.num_m_tiles * p.num_n_tiles / in_flight;
        const double t_mfast = w_bytes + (a_bytes <= l2 ? a_bytes : a_bytes * p.num_n_tiles);
        const double t_nfast = a_bytes + (w_bytes <= l2 ? w_bytes : w_bytes * (rounds_m < 1 ? 1 : rounds_m));
        p.m_fastest = t_mfast < t_nfast ? 1 : 0;
    }
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    const int slots = device_sm_count();
    const int grid = tiles < slots ? tiles : slots;
    gemm_wgmma_kernel<BN, E><<<grid, GEMM_THREADS, S::TOTAL, st>>>(tmA, tmB, tmO, tmR, p);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

// pick_bn's constants for e4m3 operands, in the order 256, 160, 128, 64. A k-block moves the same 128 bytes per operand row as
// a 16-bit one, so these start as the bf16 values below; they have not yet been fitted to per-width e4m3 timings.
static constexpr double FP8_PER_COL[4] = {1.08, 1.0, 1.03, 1.55};
static constexpr double FP8_OVERHEAD[4] = {2380.0, 1850.0, 1430.0, 780.0};

// choose the N tile (and with it the schedule, see gemm_pingpong): minimise (tiles per SM) x (per-tile time), with
//   per-tile time = per_col[bn] * bn * num_kb + overhead[bn]
// in units of one 160-wide column-k-block. Both terms are a least-squares fit (weighted by launches per call) to
// tools/bench_gemm_widths.py's per-width timings of every non-GEGLU GEMM / conv signature of a 34-row denoiser call, then
// adjusted to minimise the total of the widths chosen, on an H100 80GB HBM3 at a 700 W power limit (sw_power_cap). With
// these constants the chosen widths total 551.0 ms per call against 547.9 ms for the fastest width of every shape (563.9 ms
// with the constants fitted before the epilogue's operand passes); on a second table from another session, 563.3 against
// 559.6 ms. Under ping-pong (64, 128) the overhead is what the other warpgroup's mainloop does not hide.
// GEGLU takes the 128-wide ping-pong tile: its epilogue does the most arithmetic per column and hides best under the other
// warpgroup's mainloop.
// E4m3 (supir_gemm_fp8) has its own constants: a k-block is the same 128 bytes of each operand but twice the k-elements,
// and the k-loop is half as long for the same K (see fp8 below).
template <class E>
static int pick_bn(const GemmKernelParams& p, int force_bn) {
    const int m_tiles = p.num_m_tiles, N = p.N, num_kb = p.num_kb;
    if (force_bn == 64 || force_bn == 128 || force_bn == 160 || force_bn == 256) return force_bn;
    if (p.act == 2 && N >= 256) return 128;
    const int sms = device_sm_count();
    int best = 160;
    double best_cost = 1e30;
    const int cands[4] = {256, 160, 128, 64};
    for (int i = 0; i < 4; ++i) {
        const int bn = cands[i];
        if (bn > 64 && N <= bn / 2) continue;
        const long long tiles = (long long)m_tiles * ((N + bn - 1) / bn);
        const long long rounds = (tiles + sms - 1) / sms;
        double per_col, overhead;
        if constexpr (E::kFp8) {
            per_col = bn == 256 ? FP8_PER_COL[0] : (bn == 160 ? FP8_PER_COL[1] : (bn == 128 ? FP8_PER_COL[2] : FP8_PER_COL[3]));
            overhead = bn == 256 ? FP8_OVERHEAD[0] : (bn == 160 ? FP8_OVERHEAD[1] : (bn == 128 ? FP8_OVERHEAD[2] : FP8_OVERHEAD[3]));
        } else {
            per_col = bn == 256 ? 1.08 : (bn == 160 ? 1.0 : (bn == 128 ? 1.03 : 1.55));
            overhead = bn == 256 ? 2380.0 : (bn == 160 ? 1850.0 : (bn == 128 ? 1430.0 : 780.0));
        }
        const double cost = rounds * (per_col * bn * num_kb + overhead);
        if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
    }
    return best;
}

static int g_force_bn = 0;   // supir_set_gemm_tile_n: 0 = pick_bn's choice

// The staged epilogue needs what TMA can address: a 16-bit output and residual with 16-byte aligned base pointers and row
// strides (fp32 outputs of the text towers, odd leading dimensions and odd-address residuals take the direct stores), and
// a whole number of 32-column slabs per tile (not GEGLU at width 160, 80 output columns, which pick_bn never chooses).
// The output width must end on a 16-byte boundary (n_out % 8 == 0): a TMA store box clipped inside a 16-byte chunk
// wrote the whole chunk, past the last column, into whatever follows it in the row (a column slice's neighbours).
static bool can_stage(const GemmKernelParams& p, int bn) {
    const auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    return !p.out_f32 && (p.act != 2 || bn % 64 == 0) && p.n_out % 8 == 0 && al16(p.out) && (p.ldc * 2) % 16 == 0 &&
           (!p.residual || (al16(p.residual) && (p.ldr * 2) % 16 == 0));
}

// Tensor maps of the staged epilogue's output (tmO) and residual (tmR): boxes of 32 columns x 64 rows, 64-byte swizzle (see
// stage_off). GEMM: 2-D over [M, n_out]. Conv: 4-D over [nimg, H, W, n_out] with the output placement of the geometry (the
// interleaved sub-pixel outputs start at their offset pixel and step out_sx / out_sy pixels); the box is the 64 pixels of
// half a TH x TW patch. TMA clips the boxes at the tensor's edges.
template <class E>
static int make_epilogue_maps(GemmKernelParams& p, int bn, CUtensorMap* tmO, CUtensorMap* tmR) {
    p.staged = can_stage(p, bn) ? 1 : 0;
    if (!p.staged) return SUPIR_OK;
    using T = typename E::T;
    if (p.conv) {
        const uint32_t bw = p.TW < 64 ? p.TW : 64;
        const uint32_t box[4] = {32, bw, 64 / bw, 1};
        const uint64_t dims[4] = {(uint64_t)p.n_out, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.nimg};
        const uint64_t ost[3] = {(uint64_t)(p.ldc * p.out_sx), (uint64_t)(p.ldc * p.out_sy * p.out_W), (uint64_t)(p.ldc * p.out_H * p.out_W)};
        const T* obase = reinterpret_cast<const T*>(p.out) + ((long long)p.out_oy * p.out_W + p.out_ox) * p.ldc;
        int rc = make_tmap_16(tmO, E::kTma, obase, 4, dims, ost, box, 64);
        if (rc || !p.residual) return rc;
        const uint64_t rst[3] = {(uint64_t)p.ldr, (uint64_t)(p.ldr * p.W), (uint64_t)(p.ldr * p.W * p.H)};
        return make_tmap_16(tmR, E::kTma, p.residual, 4, dims, rst, box, 64);
    }
    const uint32_t box[2] = {32, 64};
    const uint64_t dims[2] = {(uint64_t)p.n_out, (uint64_t)p.M};
    const uint64_t ost[1] = {(uint64_t)p.ldc};
    int rc = make_tmap_16(tmO, E::kTma, p.out, 2, dims, ost, box, 64);
    if (rc || !p.residual) return rc;
    const uint64_t rst[1] = {(uint64_t)p.ldr};
    return make_tmap_16(tmR, E::kTma, p.residual, 2, dims, rst, box, 64);
}

// Picks the tile width once, then builds the W map (W: [N, K] with row stride ldw; its box is one BK x bn tile) and the
// epilogue's maps for it, and launches.
template <class E>
static int run_gemm(const CUtensorMap& tmA, const void* W, long long ldw, GemmKernelParams& p, cudaStream_t st) {
    const int bn = pick_bn<E>(p, g_force_bn);
    CUtensorMap tmB, tmO{}, tmR{};
    const uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.N};
    const uint64_t str[1] = {(uint64_t)ldw};
    const uint32_t box[2] = {(uint32_t)E::kBK, (uint32_t)bn};
    int rc = make_tmap_16(&tmB, E::kOpTma, W, 2, dims, str, box, 128, nullptr, E::kOpBytes);
    if (rc) return rc;
    rc = make_epilogue_maps<E>(p, bn, &tmO, &tmR);
    if (rc) return rc;
    if (bn == 256) return launch_gemm<256, E>(tmA, tmB, tmO, tmR, p, st);
    if (bn == 160) return launch_gemm<160, E>(tmA, tmB, tmO, tmR, p, st);
    if (bn == 128) return launch_gemm<128, E>(tmA, tmB, tmO, tmR, p, st);
    return launch_gemm<64, E>(tmA, tmB, tmO, tmR, p, st);
}

static int fill_epilogue(GemmKernelParams& p, const supir_epilogue* ep, int N) {
    p.bias = nullptr; p.rowvec = nullptr; p.rows_per_batch = 0; p.rowvec_ld = 0;
    p.residual = nullptr; p.ldr = 0; p.act = 0; p.out_f32 = 0; p.n_out = N;
    p.ln_stats = nullptr; p.ln_colsum = nullptr;
    if (ep) {
        p.ln_stats = reinterpret_cast<const float2*>(ep->ln_stats);
        p.ln_colsum = ep->ln_colsum;
        SUPIR_REQUIRE((p.ln_stats == nullptr) == (p.ln_colsum == nullptr), "epilogue: ln_stats and ln_colsum go together");
        SUPIR_REQUIRE(!p.ln_stats || (ep->act != 2 && !p.conv), "folded LayerNorm is for plain GEMM epilogues (not GEGLU, not conv)");
        SUPIR_REQUIRE(!p.ln_stats || (reinterpret_cast<uintptr_t>(ep->ln_stats) & 7) == 0, "ln_stats must be 8-byte aligned");
        p.bias = ep->bias;
        p.rowvec = ep->rowvec;
        p.rows_per_batch = ep->rows_per_batch;
        p.rowvec_ld = ep->rowvec_ld > 0 ? ep->rowvec_ld : N;
        p.residual = ep->residual;
        p.ldr = ep->ldr;
        p.act = ep->act;
        p.out_f32 = ep->out_f32;
        SUPIR_REQUIRE(p.act >= 0 && p.act <= 2, "epilogue act %d not in {0,1,2}", p.act);
        if (p.act == 2) {
            SUPIR_REQUIRE(N % 32 == 0, "GEGLU epilogue needs N %% 32 == 0 (got %d)", N);
            SUPIR_REQUIRE(!p.out_f32, "GEGLU epilogue writes bf16 only");
            p.n_out = N / 2;
        }
        if (p.residual) SUPIR_REQUIRE(p.ldr >= p.n_out, "residual ld %lld < %d", p.ldr, p.n_out);
    }
    return SUPIR_OK;
}

}  // namespace supir

using namespace supir;

extern "C" int supir_set_gemm_tile_n(int bn) {
    g_force_bn = bn;
    return SUPIR_OK;
}

template <class E>
static int gemm_impl(const char* who, const void* A, long long lda, const void* W, long long ldw, void* out, long long ldc, int M,
                     int N, int K, const supir_epilogue* ep, void* stream, const float* a_scale = nullptr,
                     const float* w_scale = nullptr) {
    SUPIR_REQUIRE(A && W && out, "%s: null pointer", who);
    SUPIR_REQUIRE(M > 0 && N > 0 && K > 0, "%s: bad shape M=%d N=%d K=%d", who, M, N, K);
    SUPIR_REQUIRE(lda % 8 == 0 && ldw % 8 == 0, "%s: lda/ldw must be multiples of 8", who);
    SUPIR_REQUIRE(lda >= K && ldw >= K, "%s: leading dims smaller than K", who);
    GemmKernelParams p{};
    p.M = M; p.N = N; p.K = K;
    p.num_m_tiles = (M + BM - 1) / BM;
    p.num_kb = (K + E::kBK - 1) / E::kBK;
    p.conv = 0;
    p.a_scale = a_scale; p.w_scale = w_scale;
    int rc = fill_epilogue(p, ep, N);
    if (rc) return rc;
    SUPIR_REQUIRE(ldc >= p.n_out, "%s: ldc %lld < output columns %d", who, ldc, p.n_out);
    p.out = out; p.ldc = ldc;
    CUtensorMap tmA;
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
    const uint64_t str[1] = {(uint64_t)lda};
    const uint32_t box[2] = {(uint32_t)E::kBK, BM};
    rc = make_tmap_16(&tmA, E::kOpTma, A, 2, dims, str, box, 128, nullptr, E::kOpBytes);
    if (rc) return rc;
    return run_gemm<E>(tmA, W, ldw, p, reinterpret_cast<cudaStream_t>(stream));
}

// E4m3: x and Wp hold e4m3 codes, with a_scale [B] (one per image) and w_scale [Cout]. Channel counts that are not a multiple
// of E::kBK read TMA's zero fill past Cin in the last chunk of every tap (its W columns are the next tap's: zero times them).
template <class E>
static int conv_geom_impl(const char* who, const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int Hin, int Win,
                          int Cin, int Cout, const supir_conv_geometry& g, const supir_epilogue* ep, void* stream,
                          const float* a_scale = nullptr, const float* w_scale = nullptr) {
    SUPIR_REQUIRE(x && Wp && out, "%s: null pointer", who);
    SUPIR_REQUIRE(B > 0 && Hin > 0 && Win > 0 && Cin > 0 && Cout > 0, "%s: bad shape", who);
    SUPIR_REQUIRE(Cin % 8 == 0 && ldx % 8 == 0 && ldx >= Cin, "%s: Cin/ldx must be multiples of 8", who);
    SUPIR_REQUIRE(g.kh >= 1 && g.kh <= 3 && g.kw >= 1 && g.kw <= 3 && (g.stride == 1 || g.stride == 2), "%s: kernel %dx%d stride %d unsupported", who, g.kh, g.kw, g.stride);
    SUPIR_REQUIRE(g.Hout > 0 && g.Wout > 0 && g.out_sy >= 1 && g.out_sx >= 1 && g.out_oy >= 0 && g.out_ox >= 0 && g.out_oy < g.out_sy &&
                  g.out_ox < g.out_sx && g.out_H >= (g.Hout - 1) * g.out_sy + g.out_oy + 1 && g.out_W >= (g.Wout - 1) * g.out_sx + g.out_ox + 1,
                  "%s: bad output geometry", who);
    const int H = g.Hout, Wd = g.Wout, ntaps = g.kh * g.kw;
    GemmKernelParams p{};
    p.conv = 1;
    p.H = H; p.W = Wd; p.Cin = Cin;
    p.ntaps_x = g.kw; p.stride = g.stride; p.off_y = g.off_y; p.off_x = g.off_x;
    p.out_sy = g.out_sy; p.out_sx = g.out_sx; p.out_oy = g.out_oy; p.out_ox = g.out_ox; p.out_H = g.out_H; p.out_W = g.out_W;
    // pixel patch per tile: TH x TW = 128 pixels; pick the shape that wastes the fewest out-of-image pixels
    {
        const int cand[5] = {16, 8, 32, 64, 128};
        long long best = -1;
        int TW = 16;
        for (int i = 0; i < 5; ++i) {
            const int tw = cand[i], th = BM / tw;
            const long long t = (long long)((Wd + tw - 1) / tw) * ((H + th - 1) / th);
            if (best < 0 || t < best) { best = t; TW = tw; }
        }
        p.TW = TW; p.TH = BM / TW;
    }
    p.tiles_x = (Wd + p.TW - 1) / p.TW;
    p.tiles_y = (H + p.TH - 1) / p.TH;
    p.num_m_tiles = B * p.tiles_x * p.tiles_y;
    p.kchunks = (Cin + E::kBK - 1) / E::kBK;
    p.num_kb = ntaps * p.kchunks;
    p.M = B * H * Wd; p.N = Cout; p.K = ntaps * Cin;
    p.nimg = B;
    p.a_scale = a_scale; p.w_scale = w_scale;
    int rc = fill_epilogue(p, ep, Cout);
    if (rc) return rc;
    SUPIR_REQUIRE(ldc >= p.n_out, "%s: ldc %lld < output columns %d", who, ldc, p.n_out);
    const bool plain_out = g.out_sy == 1 && g.out_sx == 1 && g.out_H == H && g.out_W == Wd;
    SUPIR_REQUIRE(plain_out || (!p.residual && !p.rowvec), "%s: residual / per-image vector need a plain output layout", who);
    SUPIR_REQUIRE(plain_out || (g.out_sy != 1 || g.out_sx != 1) || (g.out_H == H && g.out_W == Wd), "%s: unit-stride outputs must match the grid", who);
    p.out = out; p.ldc = ldc;
    // input [B, Hin, Win, Cin]; a tile's box covers TH x TW output pixels = every `stride`-th input pixel (elementStrides)
    CUtensorMap tmA;
    const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
    const uint64_t str[3] = {(uint64_t)ldx, (uint64_t)ldx * Win, (uint64_t)ldx * Win * Hin};
    const uint32_t box[4] = {(uint32_t)E::kBK, (uint32_t)(p.TW * g.stride), (uint32_t)(p.TH * g.stride), 1};
    const uint32_t est[4] = {1, (uint32_t)g.stride, (uint32_t)g.stride, 1};
    rc = make_tmap_16(&tmA, E::kOpTma, x, 4, dims, str, box, 128, est, E::kOpBytes);
    if (rc) return rc;
    return run_gemm<E>(tmA, Wp, p.K, p, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int supir_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldc,
                               int M, int N, int K, const supir_epilogue* ep, void* stream) {
    return gemm_impl<Bf16>("supir_gemm_bf16", A, lda, W, ldw, out, ldc, M, N, K, ep, stream);
}

extern "C" int supir_gemm_f16(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldc,
                              int M, int N, int K, const supir_epilogue* ep, void* stream) {
    return gemm_impl<F16>("supir_gemm_f16", A, lda, W, ldw, out, ldc, M, N, K, ep, stream);
}

extern "C" int supir_gemm_fp8(const void* A, long long lda, const float* a_scale, const void* W, long long ldw, const float* w_scale,
                              void* out, long long ldc, int M, int N, int K, const supir_epilogue* ep, void* stream) {
    const char* who = "supir_gemm_fp8";
    const auto al = [](const void* q, int b) { return (reinterpret_cast<uintptr_t>(q) & (b - 1)) == 0; };
    SUPIR_REQUIRE(A && W && out && a_scale && w_scale, "%s: null pointer", who);
    SUPIR_REQUIRE(K % 16 == 0 && lda % 16 == 0 && ldw % 16 == 0,
                  "%s: K, lda and ldw must be multiples of 16 (16-byte TMA row strides of e4m3), got K=%d lda=%lld ldw=%lld", who, K,
                  lda, ldw);
    SUPIR_REQUIRE(al(A, 16) && al(W, 16), "%s: A and W must be 16-byte aligned", who);
    SUPIR_REQUIRE(al(a_scale, 4) && al(w_scale, 4), "%s: scales must be 4-byte aligned fp32", who);
    SUPIR_REQUIRE(al(out, 2) && (!ep || !ep->residual || al(ep->residual, 2)), "%s: out / residual must be 2-byte aligned bf16", who);
    SUPIR_REQUIRE(!ep || (!ep->out_f32 && !ep->ln_stats && !ep->ln_colsum && !ep->rowvec),
                  "%s: the FP8 epilogue writes bf16 and takes bias / residual / GEGLU only (no out_f32, ln_stats, rowvec)", who);
    return gemm_impl<E4m3>(who, A, lda, W, ldw, out, ldc, M, N, K, ep, stream, a_scale, w_scale);
}

extern "C" int supir_conv_geom_bf16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int Hin, int Win,
                                    int Cin, int Cout, const supir_conv_geometry* geom, const supir_epilogue* ep, void* stream) {
    SUPIR_REQUIRE(geom, "supir_conv_geom_bf16: null geometry");
    return conv_geom_impl<Bf16>("supir_conv_geom_bf16", x, ldx, Wp, out, ldc, B, Hin, Win, Cin, Cout, *geom, ep, stream);
}

extern "C" int supir_conv_geom_f16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int Hin, int Win,
                                   int Cin, int Cout, const supir_conv_geometry* geom, const supir_epilogue* ep, void* stream) {
    SUPIR_REQUIRE(geom, "supir_conv_geom_f16: null geometry");
    return conv_geom_impl<F16>("supir_conv_geom_f16", x, ldx, Wp, out, ldc, B, Hin, Win, Cin, Cout, *geom, ep, stream);
}

// 3x3, stride 1, pad 1
static supir_conv_geometry conv3x3_geometry(int H, int Wd) {
    supir_conv_geometry g{};
    g.kh = g.kw = 3; g.stride = 1; g.off_y = g.off_x = -1;
    g.Hout = H; g.Wout = Wd;
    g.out_sy = g.out_sx = 1; g.out_oy = g.out_ox = 0; g.out_H = H; g.out_W = Wd;
    return g;
}

extern "C" int supir_conv3x3_bf16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int H,
                                  int Wd, int Cin, int Cout, const supir_epilogue* ep, void* stream) {
    return conv_geom_impl<Bf16>("supir_conv3x3_bf16", x, ldx, Wp, out, ldc, B, H, Wd, Cin, Cout, conv3x3_geometry(H, Wd), ep, stream);
}

extern "C" int supir_conv3x3_f16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int H,
                                 int Wd, int Cin, int Cout, const supir_epilogue* ep, void* stream) {
    return conv_geom_impl<F16>("supir_conv3x3_f16", x, ldx, Wp, out, ldc, B, H, Wd, Cin, Cout, conv3x3_geometry(H, Wd), ep, stream);
}

extern "C" int supir_conv3x3_fp8(const void* x, long long ldx, const float* x_scale, const void* Wp, const float* w_scale, void* out,
                                 long long ldc, int B, int H, int Wd, int Cin, int Cout, const supir_epilogue* ep, void* stream) {
    const char* who = "supir_conv3x3_fp8";
    const auto al = [](const void* q, int b) { return (reinterpret_cast<uintptr_t>(q) & (b - 1)) == 0; };
    SUPIR_REQUIRE(x && Wp && out && x_scale && w_scale, "%s: null pointer", who);
    SUPIR_REQUIRE(B > 0 && H > 0 && Wd > 0 && Cin > 0 && Cout > 0, "%s: bad shape B=%d H=%d W=%d Cin=%d Cout=%d", who, B, H, Wd, Cin,
                  Cout);
    SUPIR_REQUIRE(Cin % 16 == 0 && ldx % 16 == 0 && ldx >= Cin,
                  "%s: Cin and ldx must be multiples of 16 (16-byte TMA strides of e4m3), ldx >= Cin; got Cin=%d ldx=%lld", who, Cin, ldx);
    SUPIR_REQUIRE(al(x, 16) && al(Wp, 16), "%s: x and Wp must be 16-byte aligned", who);
    SUPIR_REQUIRE(al(x_scale, 4) && al(w_scale, 4), "%s: scales must be 4-byte aligned fp32", who);
    SUPIR_REQUIRE(al(out, 2) && (!ep || !ep->residual || al(ep->residual, 2)), "%s: out / residual must be 2-byte aligned bf16", who);
    SUPIR_REQUIRE(!ep || (!ep->out_f32 && !ep->ln_stats && !ep->ln_colsum && ep->act != 2),
                  "%s: the FP8 conv epilogue writes bf16 and takes bias / rowvec / residual / SiLU only (no out_f32, ln_stats, GEGLU)",
                  who);
    return conv_geom_impl<E4m3>(who, x, ldx, Wp, out, ldc, B, H, Wd, Cin, Cout, conv3x3_geometry(H, Wd), ep, stream, x_scale, w_scale);
}
