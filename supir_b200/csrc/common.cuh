// supir_b200 — sm_90a device helpers: mbarrier and TMA inline-PTX wrappers (wgmma wrappers: wgmma.cuh).
// Every kernel in this directory is written for H100 (sm_90a) only; there is no other target.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace supir {

// ---------------------------------------------------------------------------------------------
// error plumbing shared by all translation units (defined in api.cu)
// ---------------------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);  // bumps the counter behind supir_launch_count()
int device_sm_count();
int current_device_slot();   // cudaGetDevice() clamped to [0, 63]: index of the per-device caches

// Tensor map of 16-bit elements, or of `elem_bytes`-byte ones (defined in gemm.cu): dims / strides innermost first, strides in
// elements; `swizzle` in bytes; `elem_strides` (null: all 1) are TMA traversal strides. Rejects base addresses and strides TMA
// cannot take.
int make_tmap_16(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_elems, const uint32_t* box, int swizzle = 128, const uint32_t* elem_strides = nullptr,
                 int elem_bytes = 2);

#define SUPIR_OK 0
#define SUPIR_ERR_INVALID -1
#define SUPIR_ERR_CUDA -2
#define SUPIR_ERR_UNSUPPORTED -3

#define SUPIR_CHECK_CUDA(expr)                                                              \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess)                                                              \
            return supir::set_error(SUPIR_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,          \
                                    cudaGetErrorString(_e), __FILE__, __LINE__);            \
    } while (0)

#define SUPIR_REQUIRE(cond, ...)                                                            \
    do {                                                                                    \
        if (!(cond)) return supir::set_error(SUPIR_ERR_INVALID, __VA_ARGS__);               \
    } while (0)

// ---------------------------------------------------------------------------------------------
// small device utilities
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
    __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(t);
}

__device__ __forceinline__ float f16_round(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
    __half2 t = __floats2half2_rn(lo, hi);     // cvt.rn.f16x2.f32
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t u) {
    __half2 t = *reinterpret_cast<__half2*>(&u);
    return __half22float2(t);
}

// ---------------------------------------------------------------------------------------------
// 16-bit storage element types. The diffusion-network kernels are templated on one of these; everything that is not
// storage (accumulators, statistics, softmax) stays fp32 in both. The instantiation with Bf16 is the original bf16 kernel.
//   round       : fp32 -> nearest storage value, back as fp32 (the points where autocast rounds an intermediate tensor)
//   pack2/unpack2: two fp32 <-> one 32-bit register of two storage values (round to nearest even)
//   from_f/to_f : scalar conversions; bits: the raw 16 bits
//   kF16        : selects the wgmma operand types (.f16.f16 instead of .bf16.bf16, see wgmma.cuh)
//   kTma        : TMA data type of the 16-bit tensor maps (output, residual; and the GEMM operands unless kFp8)
// GEMM operand side (gemm.cu): the operands are the storage type itself, except under E4m3 below.
//   kFp8        : e4m3 operands (.e4m3.e4m3, m64nNk32) with per-row / per-column fp32 scales applied in the epilogue
//   kOpTma      : TMA data type of the operand maps; kOpBytes: bytes per operand element
//   kBK         : operand elements per k-block = one 128-byte swizzled row (64 16-bit or 128 e4m3 elements)
// ---------------------------------------------------------------------------------------------
struct Bf16 {
    using T = __nv_bfloat16;
    static constexpr bool kF16 = false;
    static constexpr CUtensorMapDataType kTma = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    static constexpr bool kFp8 = false;
    static constexpr CUtensorMapDataType kOpTma = kTma;
    static constexpr int kOpBytes = 2;
    static constexpr int kBK = 64;
    static __device__ __forceinline__ float round(float v) { return bf16_round(v); }
    static __device__ __forceinline__ uint32_t pack2(float lo, float hi) { return pack_bf16x2(lo, hi); }
    static __device__ __forceinline__ float2 unpack2(uint32_t u) { return unpack_bf16x2(u); }
    static __device__ __forceinline__ T from_f(float v) { return __float2bfloat16_rn(v); }
    static __device__ __forceinline__ float to_f(T v) { return __bfloat162float(v); }
    static __device__ __forceinline__ uint32_t bits(T v) { return __bfloat16_as_ushort(v); }
};
struct F16 {
    using T = __half;
    static constexpr bool kF16 = true;
    static constexpr CUtensorMapDataType kTma = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    static constexpr bool kFp8 = false;
    static constexpr CUtensorMapDataType kOpTma = kTma;
    static constexpr int kOpBytes = 2;
    static constexpr int kBK = 64;
    static __device__ __forceinline__ float round(float v) { return f16_round(v); }
    static __device__ __forceinline__ uint32_t pack2(float lo, float hi) { return pack_f16x2(lo, hi); }
    static __device__ __forceinline__ float2 unpack2(uint32_t u) { return unpack_f16x2(u); }
    static __device__ __forceinline__ T from_f(float v) { return __float2half_rn(v); }
    static __device__ __forceinline__ float to_f(T v) { return __half2float(v); }
    static __device__ __forceinline__ uint32_t bits(T v) { return __half_as_ushort(v); }
};

// FP8 linear layers (supir_gemm_fp8): e4m3 operands, bf16 storage everywhere else. Every epilogue rounding point is bf16's.
struct E4m3 : Bf16 {
    static constexpr bool kFp8 = true;
    static constexpr CUtensorMapDataType kOpTma = CU_TENSOR_MAP_DATA_TYPE_UINT8;
    static constexpr int kOpBytes = 1;
    static constexpr int kBK = 128;
};

// Row quantization to e4m3 (quantize_rows, LayerNorm-quant): scale = amax / 448 (1 for an all-zero row) and
// code = RNE(x * (448 / amax)), with the two divisions IEEE-rounded: the codes and scales are those of
// (x * inv).to(torch.float8_e4m3fn) on the same fp32 values. |x * inv| <= 448 up to one ulp, which rounds to 448: the
// saturating conversion never saturates a value torch would not round to 448 as well.
__device__ __forceinline__ void e4m3_row_scale(float amax, float& scale, float& inv) {
    scale = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
    inv = amax > 0.f ? __fdiv_rn(448.f, amax) : 1.f;
}
// four fp32 -> four e4m3 codes in one 32-bit word (first value in the low byte)
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
    return (lo & 0xFFFFu) | (hi << 16);
}

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// erf-form GELU — F.gelu default used by GEGLU (reference sgm/modules/attention.py:91):  gelu(g) = g/2 + |g|/2 * erf(|g|/sqrt2).
// erf via Abramowitz-Stegun 7.1.26 (abs err <= 1.5e-7, far below the bf16 rounding of the result) with 1/sqrt2 folded
// into the constants: 2 MUFU (rcp, ex2) + 7 FFMA + 4 FMUL, branch-free, where libdevice erff takes ~40 instructions
// with a slow path.
__device__ __forceinline__ float gelu_erf_f(float g) {
    const float ag = fabsf(g);
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.2316418882f, ag, 1.0f)));   // 1 / (1 + p |g| / sqrt2)
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    poly *= t;
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(g * g * -0.7213475204f));          // exp(-g^2 / 2)
    const float erf_abs = fmaf(-poly, e, 1.0f);                                          // erf(|g| / sqrt2)
    const float h = 0.5f * g;
    return fmaf(fabsf(h), erf_abs, h);
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)   // suspend-time hint: the hardware parks the thread instead of spinning
        : "memory");
    return ok != 0;
}
// non-blocking probe (no suspend): for the MMA issuer's event loop
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads; completion is signalled on an mbarrier (complete_tx::bytes)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}


// TMA stores (shared -> global, bulk async group); the issuing thread tracks completion with commit / wait_group
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// signal a named barrier without waiting on it (the waiting side uses named_bar_sync with the same thread count)
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// 2^x on the FMA / ALU pipes (no MUFU). x is clamped at -126 (result 2^-126 ~ 0 for anything below, including the -inf
// of masked keys): Cody-Waite split x = n + f (round-down add of the 1.5*2^23 magic constant), degree-3 minimax
// polynomial for 2^f on [0,1) (max rel. error 8.8e-5 = 2^-13.5, far below the bf16 rounding of P at 2^-9), exponent
// reinserted with one integer shift-add.
__device__ __forceinline__ float ex2_emulated(float x) {
    const float kMagic = 12582912.0f;                       // 1.5 * 2^23: x + magic has ulp 1, floor(x) lands in the low mantissa bits
    x = fmaxf(x, -126.0f);
    const float xr = __fadd_rd(x, kMagic);                  // magic + floor(x)
    const float xf = __fadd_rn(xr, -kMagic);                // floor(x), exact
    const float fr = __fadd_rn(x, -xf);                     // x - floor(x) in [0, 1), exact
    float p = fmaf(0.077119089663028717041015625f, fr, 0.227564394474029541015625f);
    p = fmaf(p, fr, 0.695146143436431884765625f);
    p = fmaf(p, fr, 1.0f);                                  // 2^f in [1, 2]
    // bits(magic + n) = 0x4B400000 + n: the low 9 bits of the constant are zero, so << 23 leaves n in the exponent field
    return __uint_as_float(__float_as_uint(p) + (__float_as_uint(xr) << 23));
}

}  // namespace supir
