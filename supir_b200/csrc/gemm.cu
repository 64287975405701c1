// supir_b200 — K2/K3/K4 of SURVEY.md §2a: Linear, conv1x1 and conv3x3 (implicit GEMM) on Hopper wgmma.
//
//   out[m, n] = epilogue( sum_k A[m, k] * W[n, k] )          bf16 x bf16 -> fp32 (registers) -> bf16/fp32
//
// Replaces, on the sampling path of the reference: nn.Linear (sgm/modules/attention.py:213-218,87,106,587,611),
// nn.Conv2d 1x1 (openaimodel.py:317, SUPIR_v0.py:48,87, model.py:124-126,164-175) and nn.Conv2d 3x3 stride 1 pad 1
// (openaimodel.py:263,300-307; SUPIR_v0.py:79,82-83; model.py:108-117 ...).
//
// Design (one persistent CTA per SM, 384 threads = three warpgroups, warp-specialised):
//   warpgroup 0, thread 0 : TMA producer.  A tile = 128 rows x 64 k (bf16, 128B-swizzled), W tile = BN rows x 64 k.
//                   GEMM mode: A is a 2-D tensor map over [M, K].
//                   CONV mode: A is a 4-D tensor map over the NHWC activation [B, H, W, C]; the tile's 128 rows are a
//                   TH x TW pixel patch and the k-loop runs over (tap, 64-channel chunk); the tap shift is applied to the
//                   TMA coordinates, and TMA's out-of-bounds zero fill IS the conv padding (no im2col buffer).
//   warpgroups 1, 2       : wgmma consumers, rows [0, 64) and [64, 128) of the tile (m64nBNk16, fp32 accumulators in
//                   registers, one wgmma group kept in flight); then the epilogue straight from the accumulator fragment:
//                   +bias, +per-batch vector (timestep embedding), folded LayerNorm, SiLU / GEGLU, bf16 round, +residual,
//                   bf16 or fp32 stores. The producer keeps filling the shared-memory ring for the next tile meanwhile.
// Pipeline: smem full/empty mbarrier ring (TMA <-> wgmma).
#include "common.cuh"
#include "supir_b200.h"
#include "wgmma.cuh"

#include <cstdlib>
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
    const __nv_bfloat16* residual;
    long long ldr;
    int act;
    void* out;
    long long ldc;
    int out_f32;
    int n_out;            // valid output columns (N or N/2 for GEGLU)
    int nimg;             // conv mode: number of images
    const float2* ln_stats;  // per-row (rstd, mean * rstd) of A: LayerNorm folded into the epilogue (see supir_epilogue), or null
    const float* ln_colsum;  // [N] row sums of the (gamma-scaled) weight matrix
};

template <int BN>
struct GemmSmem {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (192 * 1024) / STAGE_BYTES > 8 ? 8 : (192 * 1024) / STAGE_BYTES;   // 4..8 stages, <= 192 KB
    static constexpr int BAR_BYTES = 256;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + BAR_BYTES + 1024;  // +1024 alignment slack
};

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
    if constexpr (BN == 256) wgmma_ss_n256(d, da, db, scale_d);
    else if constexpr (BN == 160) wgmma_ss_n160(d, da, db, scale_d);
    else if constexpr (BN == 128) wgmma_ss_n128(d, da, db, scale_d);
    else wgmma_ss_n64(d, da, db, scale_d);
}

// two adjacent output columns (n, n + 1) of one row; `n1ok`: column n + 1 exists
__device__ __forceinline__ void store_pair(const GemmKernelParams& p, long long grow, int n, float v0, float v1, bool n1ok) {
    if (p.out_f32) {
        float* dst = reinterpret_cast<float*>(p.out) + grow * p.ldc + n;
        if (n1ok && ((reinterpret_cast<uintptr_t>(dst) & 7) == 0)) { *reinterpret_cast<float2*>(dst) = make_float2(v0, v1); }
        else { dst[0] = v0; if (n1ok) dst[1] = v1; }
    } else {
        __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out) + grow * p.ldc + n;
        if (n1ok && ((reinterpret_cast<uintptr_t>(dst) & 3) == 0)) { *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(v0, v1); }
        else { dst[0] = __float2bfloat16_rn(v0); if (n1ok) dst[1] = __float2bfloat16_rn(v1); }
    }
}
__device__ __forceinline__ float2 load_res_pair(const GemmKernelParams& p, long long grow, int n, bool n1ok) {
    const __nv_bfloat16* src = p.residual + grow * p.ldr + n;
    if (n1ok && ((reinterpret_cast<uintptr_t>(src) & 3) == 0)) return unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(src)));
    return make_float2(__bfloat162float(src[0]), n1ok ? __bfloat162float(src[1]) : 0.f);
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKernelParams p) {
    using S = GemmSmem<BN>;
    constexpr int STAGES = S::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * S::A_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES);   // [STAGES]
    uint64_t* empty_bar = full_bar + STAGES;                                              // [STAGES]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.num_m_tiles * p.num_n_tiles;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
        }
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
                const int mt = p.m_fastest ? tile % p.num_m_tiles : tile / p.num_n_tiles;
                const int nt = p.m_fastest ? tile / p.num_m_tiles : tile % p.num_n_tiles;
                int b = 0, y0 = 0, x0 = 0;
                if (p.conv) {
                    const int per_img = p.tiles_x * p.tiles_y;
                    b = mt / per_img;
                    const int r = mt % per_img;
                    y0 = (r / p.tiles_x) * p.TH;
                    x0 = (r % p.tiles_x) * p.TW;
                }
                const int bn0 = nt * BN;
                // conv mode walks (tap row, tap column, 64-channel chunk) with counters: no division in the per-k-block path
                int cc = 0, tx = 0, ty = 0, wcol = 0;
                const int ax0 = x0 * p.stride + p.off_x, ay0 = y0 * p.stride + p.off_y;
                for (int kb = 0; kb < p.num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], S::STAGE_BYTES);
                    uint8_t* sa = smem_a + stage * S::A_BYTES;
                    uint8_t* sb = smem_b + stage * S::B_BYTES;
                    if (p.conv) {
                        tma_load_4d(sa, &tmA, &full_bar[stage], cc * BK, ax0 + tx, ay0 + ty, b);
                        tma_load_2d(sb, &tmB, &full_bar[stage], wcol + cc * BK, bn0);
                        if (++cc == p.kchunks) {                       // next tap: W columns advance by Cin
                            cc = 0;
                            wcol += p.Cin;
                            if (++tx == p.ntaps_x) { tx = 0; ++ty; }
                        }
                    } else {
                        tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, mt * BM);
                        tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, bn0);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ===================== wgmma consumers + epilogue (warpgroups 1, 2) =====================
        const int wg = (warp - 4) >> 2;                       // rows [64 wg, 64 wg + 64) of the tile
        const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // accumulator rows r_lo and r_lo + 8
        const int cq = 2 * (lane & 3);                        // first of the two columns this thread holds per 8-column block
        float acc[BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int mt = p.m_fastest ? tile % p.num_m_tiles : tile / p.num_n_tiles;
            const int nt = p.m_fastest ? tile / p.num_m_tiles : tile % p.num_n_tiles;
            int prev = -1;
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem_a + stage * S::A_BYTES + wg * 64 * 128);
                const uint32_t b_addr = smem_u32(smem_b + stage * S::B_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)       // 16 k-elements = 32 bytes inside the 128B swizzle row
                    wgmma_tile<BN>(acc, wgmma_desc_sw128(a_addr + 32 * k), wgmma_desc_sw128(b_addr + 32 * k), (kb | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();                         // the previous k-block's group has retired: its slot is free
                if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_fence_operands(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);

            // ---------------- epilogue, from the accumulator fragment ----------------
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row_in_tile = r_lo + 8 * h;
                long long grow;
                int batch_idx;
                bool row_ok;
                if (p.conv) {
                    const int per_img = p.tiles_x * p.tiles_y;
                    const int b = mt / per_img;
                    const int r = mt % per_img;
                    const int y = (r / p.tiles_x) * p.TH + row_in_tile / p.TW;
                    const int x = (r % p.tiles_x) * p.TW + row_in_tile % p.TW;
                    row_ok = (y < p.H) && (x < p.W) && (b < p.nimg);
                    grow = ((long long)b * p.out_H + (long long)y * p.out_sy + p.out_oy) * p.out_W + (long long)x * p.out_sx + p.out_ox;
                    batch_idx = b;
                } else {
                    grow = (long long)mt * BM + row_in_tile;
                    row_ok = grow < p.M;
                    batch_idx = p.rows_per_batch > 0 ? (int)(grow / p.rows_per_batch) : 0;
                }
                if (!row_ok) continue;
                const float* rv = p.rowvec ? p.rowvec + (long long)batch_idx * p.rowvec_ld : nullptr;
                if (p.act == 2) {
                    // GEGLU: accumulator columns come in groups of 32 = [16 value | 16 gate]; this thread holds value column
                    // 8 b + cq (+1) of group g in block 4 g + b and its gate 16 columns later in block 4 g + b + 2
#pragma unroll
                    for (int g = 0; g < BN / 32; ++g) {
                        if (nt * BN + g * 32 >= p.N) break;
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            const int nv = nt * BN + g * 32 + b * 8 + cq;
                            float xv0 = acc[4 * (4 * g + b) + 2 * h], xv1 = acc[4 * (4 * g + b) + 2 * h + 1];
                            float gv0 = acc[4 * (4 * g + b + 2) + 2 * h], gv1 = acc[4 * (4 * g + b + 2) + 2 * h + 1];
                            if (p.bias) {
                                xv0 += __ldg(p.bias + nv); xv1 += __ldg(p.bias + nv + 1);
                                gv0 += __ldg(p.bias + nv + 16); gv1 += __ldg(p.bias + nv + 17);
                            }
                            if (rv) {
                                xv0 += __ldg(rv + nv); xv1 += __ldg(rv + nv + 1);
                                gv0 += __ldg(rv + nv + 16); gv1 += __ldg(rv + nv + 17);
                            }
                            float o0 = bf16_round(bf16_round(xv0) * bf16_round(gelu_erf_f(bf16_round(gv0))));
                            float o1 = bf16_round(bf16_round(xv1) * bf16_round(gelu_erf_f(bf16_round(gv1))));
                            const int oc = (nt * BN) / 2 + g * 16 + b * 8 + cq;
                            if (p.residual) {
                                const float2 r = load_res_pair(p, grow, oc, true);
                                o0 += r.x; o1 += r.y;
                            }
                            store_pair(p, grow, oc, o0, o1, true);
                        }
                    }
                } else {
                    float ln_rs = 1.f, ln_nm = 0.f;
                    if (p.ln_stats) { const float2 st = __ldg(p.ln_stats + grow); ln_rs = st.x; ln_nm = st.y; }
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j) {
                        const int n = nt * BN + 8 * j + cq;
                        if (n >= p.N) break;
                        const bool n1ok = n + 1 < p.N;
                        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                        if (p.ln_stats) {
                            v0 = fmaf(v0, ln_rs, -ln_nm * __ldg(p.ln_colsum + n));
                            if (n1ok) v1 = fmaf(v1, ln_rs, -ln_nm * __ldg(p.ln_colsum + n + 1));
                        }
                        if (p.bias) { v0 += __ldg(p.bias + n); if (n1ok) v1 += __ldg(p.bias + n + 1); }
                        if (rv) { v0 += __ldg(rv + n); if (n1ok) v1 += __ldg(rv + n + 1); }
                        if (p.act == 1) { v0 = silu_f(bf16_round(v0)); v1 = silu_f(bf16_round(v1)); }
                        if (p.residual) {
                            const float2 r = load_res_pair(p, grow, n, n1ok);
                            if (p.out_f32) { v0 += r.x; v1 += r.y; }
                            else { v0 = bf16_round(v0) + r.x; v1 = bf16_round(v1) + r.y; }
                        }
                        store_pair(p, grow, n, v0, v1, n1ok);
                    }
                }
            }
        }
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

// rank-N bf16 tensor map with 128B swizzle; dims/strides innermost first; strides in ELEMENTS for dims 1..rank-1
int make_tmap_bf16_sw(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                      const uint32_t* box, int swizzle_bytes) {
    PFN_tmapEncodeTiled fn = get_encode_fn();
    if (!fn) return set_error(SUPIR_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
    }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_elems[i] * 2;
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
        return set_error(SUPIR_ERR_INVALID, "TMA base address %p is not 16-byte aligned", base);
    for (int i = 0; i + 1 < rank; ++i)
        if (gstr[i] % 16 != 0) return set_error(SUPIR_ERR_INVALID, "TMA stride %d (%llu B) not a multiple of 16", i,
                                                 (unsigned long long)gstr[i]);
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                  : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(SUPIR_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return SUPIR_OK;
}

int make_tmap_bf16(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                   const uint32_t* box) {
    return make_tmap_bf16_sw(m, base, rank, dims, strides_elems, box, 128);
}

// same with traversal strides (elementStrides): the box spans box[i] tensor elements of dimension i and delivers every
// elem_strides[i]-th of them, densely packed (a stride-2 convolution's input patch)
int make_tmap_bf16_strided(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                           const uint32_t* box, const uint32_t* elem_strides) {
    PFN_tmapEncodeTiled fn = get_encode_fn();
    if (!fn) return set_error(SUPIR_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = elem_strides[i]; }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_elems[i] * 2;
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(SUPIR_ERR_INVALID, "TMA base address %p is not 16-byte aligned", base);
    for (int i = 0; i + 1 < rank; ++i)
        if (gstr[i] % 16 != 0) return set_error(SUPIR_ERR_INVALID, "TMA stride %d (%llu B) not a multiple of 16", i, (unsigned long long)gstr[i]);
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(SUPIR_ERR_CUDA, "cuTensorMapEncodeTiled (strided) failed with CUresult %d", (int)r);
    return SUPIR_OK;
}

// current device, clamped into the per-device caches below (function attributes and SM counts are per device)
int current_device_slot() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev < 0 ? 0 : (dev > 63 ? 63 : dev);
}

int device_sm_count() {
    static int sms[64] = {};
    const int d = current_device_slot();
    if (sms[d] == 0) {
        cudaDeviceGetAttribute(&sms[d], cudaDevAttrMultiProcessorCount, d);
        if (sms[d] <= 0) sms[d] = 132;
    }
    return sms[d];
}

extern int g_force_bn;

template <int BN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmKernelParams p, cudaStream_t st) {
    using S = GemmSmem<BN>;
    static bool attr_set[64] = {};
    const int dslot = current_device_slot();
    if (!attr_set[dslot]) {
        SUPIR_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
        attr_set[dslot] = true;
    }
    p.num_n_tiles = (p.N + BN - 1) / BN;
    p.nimg = p.conv ? (int)(p.M / ((long long)p.H * p.W)) : 0;
    {
        // tile order that minimises HBM traffic under a simple L2 model (50 MB of L2 on H100): the CTAs running together
        // (one round) either share a W tile (m-fastest; A is re-streamed once per n-tile unless it fits L2) or share an A tile
        // (n-fastest; W is re-streamed once per round of m-tiles unless it fits L2)
        const double l2 = 50e6;
        const double a_bytes = 2.0 * p.M * (p.conv ? p.Cin : p.K), w_bytes = 2.0 * p.N * p.K;
        const double rounds_m = (double)p.num_m_tiles * p.num_n_tiles / device_sm_count();
        const double t_mfast = w_bytes + (a_bytes <= l2 ? a_bytes : a_bytes * p.num_n_tiles);
        const double t_nfast = a_bytes + (w_bytes <= l2 ? w_bytes : w_bytes * (rounds_m < 1 ? 1 : rounds_m));
        p.m_fastest = t_mfast < t_nfast ? 1 : 0;
    }
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    const int slots = device_sm_count();
    const int grid = tiles < slots ? tiles : slots;
    gemm_wgmma_kernel<BN><<<grid, GEMM_THREADS, S::TOTAL, st>>>(tmA, tmB, p);
    count_launch();
    SUPIR_CHECK_CUDA(cudaGetLastError());
    return SUPIR_OK;
}

// choose the N tile: minimise (rounds over the SMs) x (per-tile time). 160 divides every channel count of SUPIR
// (320..10240) exactly; 256 has the best shared-memory traffic per flop; narrow tiles fill the machine for small M.
static int pick_bn(const GemmKernelParams& p, int force_bn) {
    const int m_tiles = p.num_m_tiles, N = p.N, num_kb = p.num_kb;
    if (force_bn == 64 || force_bn == 128 || force_bn == 160 || force_bn == 256) return force_bn;
    const int sms = device_sm_count();
    int best = 128;
    double best_cost = 1e30;
    const int cands[4] = {256, 160, 128, 64};
    for (int i = 0; i < 4; ++i) {
        const int bn = cands[i];
        if (bn > 64 && N <= bn / 2) continue;
        const long long tiles = (long long)m_tiles * ((N + bn - 1) / bn);
        const long long rounds = (tiles + sms - 1) / sms;
        // MMA time of a tile ~ bn * num_kb, with a per-column penalty for narrow tiles (each k-block re-reads the whole A
        // tile from shared memory for fewer columns); plus a per-tile overhead (pipeline fill + epilogue, which does not
        // overlap the next tile's MMAs) of ~6 k-blocks of a 256-wide tile. Relative estimates, not measurements.
        const double per_col = bn == 256 ? 1.0 : (bn == 160 ? 1.1 : (bn == 128 ? 1.2 : 1.6));
        const double tile_cost = bn * per_col * num_kb + 256.0 * 6.0;
        const double cost = rounds * tile_cost;
        if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
    }
    return best;
}

int g_force_bn = 0;

static int run_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmKernelParams& p, cudaStream_t st) {
    const int bn = pick_bn(p, g_force_bn);
    if (bn == 256) return launch_gemm<256>(tmA, tmB, p, st);
    if (bn == 160) return launch_gemm<160>(tmA, tmB, p, st);
    if (bn == 128) return launch_gemm<128>(tmA, tmB, p, st);
    return launch_gemm<64>(tmA, tmB, p, st);
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
        p.residual = reinterpret_cast<const __nv_bfloat16*>(ep->residual);
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

extern "C" int supir_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldc,
                               int M, int N, int K, const supir_epilogue* ep, void* stream) {
    SUPIR_REQUIRE(A && W && out, "supir_gemm_bf16: null pointer");
    SUPIR_REQUIRE(M > 0 && N > 0 && K > 0, "supir_gemm_bf16: bad shape M=%d N=%d K=%d", M, N, K);
    SUPIR_REQUIRE(lda % 8 == 0 && ldw % 8 == 0, "supir_gemm_bf16: lda/ldw must be multiples of 8");
    SUPIR_REQUIRE(lda >= K && ldw >= K, "supir_gemm_bf16: leading dims smaller than K");
    GemmKernelParams p{};
    p.M = M; p.N = N; p.K = K;
    p.num_m_tiles = (M + BM - 1) / BM;
    p.num_kb = (K + BK - 1) / BK;
    p.conv = 0;
    int rc = fill_epilogue(p, ep, N);
    if (rc) return rc;
    SUPIR_REQUIRE(ldc >= p.n_out, "supir_gemm_bf16: ldc %lld < output columns %d", ldc, p.n_out);
    p.out = out; p.ldc = ldc;
    const int bn = pick_bn(p, g_force_bn);
    CUtensorMap tmA, tmB;
    {
        const uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
        const uint64_t str[1] = {(uint64_t)lda};
        const uint32_t box[2] = {BK, BM};
        rc = make_tmap_bf16(&tmA, A, 2, dims, str, box);
        if (rc) return rc;
    }
    {
        const uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
        const uint64_t str[1] = {(uint64_t)ldw};
        const uint32_t box[2] = {BK, (uint32_t)bn};
        rc = make_tmap_bf16(&tmB, W, 2, dims, str, box);
        if (rc) return rc;
    }
    return run_gemm(tmA, tmB, p, reinterpret_cast<cudaStream_t>(stream));
}

static int conv_geom_impl(const char* who, const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int Hin, int Win,
                          int Cin, int Cout, const supir_conv_geometry& g, const supir_epilogue* ep, void* stream) {
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
    p.kchunks = (Cin + BK - 1) / BK;
    p.num_kb = ntaps * p.kchunks;
    p.M = B * H * Wd; p.N = Cout; p.K = ntaps * Cin;
    int rc = fill_epilogue(p, ep, Cout);
    if (rc) return rc;
    SUPIR_REQUIRE(ldc >= p.n_out, "%s: ldc %lld < output columns %d", who, ldc, p.n_out);
    const bool plain_out = g.out_sy == 1 && g.out_sx == 1 && g.out_H == H && g.out_W == Wd;
    SUPIR_REQUIRE(plain_out || (!p.residual && !p.rowvec), "%s: residual / per-image vector need a plain output layout", who);
    SUPIR_REQUIRE(plain_out || (g.out_sy != 1 || g.out_sx != 1) || (g.out_H == H && g.out_W == Wd), "%s: unit-stride outputs must match the grid", who);
    p.out = out; p.ldc = ldc;
    const int bn = pick_bn(p, g_force_bn);
    CUtensorMap tmA, tmB;
    {
        // input [B, Hin, Win, Cin]; a tile's box covers TH x TW output pixels = every `stride`-th input pixel (elementStrides)
        const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
        const uint64_t str[3] = {(uint64_t)ldx, (uint64_t)ldx * Win, (uint64_t)ldx * Win * Hin};
        const uint32_t box[4] = {BK, (uint32_t)(p.TW * g.stride), (uint32_t)(p.TH * g.stride), 1};
        const uint32_t est[4] = {1, (uint32_t)g.stride, (uint32_t)g.stride, 1};
        rc = make_tmap_bf16_strided(&tmA, x, 4, dims, str, box, est);
        if (rc) return rc;
    }
    {
        const uint64_t dims[2] = {(uint64_t)(ntaps * Cin), (uint64_t)Cout};
        const uint64_t str[1] = {(uint64_t)(ntaps * Cin)};
        const uint32_t box[2] = {BK, (uint32_t)bn};
        rc = make_tmap_bf16(&tmB, Wp, 2, dims, str, box);
        if (rc) return rc;
    }
    return run_gemm(tmA, tmB, p, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int supir_conv_geom_bf16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int Hin, int Win,
                                    int Cin, int Cout, const supir_conv_geometry* geom, const supir_epilogue* ep, void* stream) {
    SUPIR_REQUIRE(geom, "supir_conv_geom_bf16: null geometry");
    return conv_geom_impl("supir_conv_geom_bf16", x, ldx, Wp, out, ldc, B, Hin, Win, Cin, Cout, *geom, ep, stream);
}

extern "C" int supir_conv3x3_bf16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int H,
                                  int Wd, int Cin, int Cout, const supir_epilogue* ep, void* stream) {
    supir_conv_geometry g{};
    g.kh = g.kw = 3; g.stride = 1; g.off_y = g.off_x = -1;
    g.Hout = H; g.Wout = Wd;
    g.out_sy = g.out_sx = 1; g.out_oy = g.out_ox = 0; g.out_H = H; g.out_W = Wd;
    return conv_geom_impl("supir_conv3x3_bf16", x, ldx, Wp, out, ldc, B, H, Wd, Cin, Cout, g, ep, stream);
}
