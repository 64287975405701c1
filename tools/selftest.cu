// Standalone GPU self-test + micro-benchmark for libsupir_b200.so (no Python, no torch).
// Used during bring-up under gpurun:   timeout 120 tools/selftest gemm|conv|perf|all
// Each check compares the C-ABI kernel with a plain fp32 CPU loop on bf16-rounded inputs.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "supir_b200.h"

#define CK(x)                                                                                  \
    do {                                                                                       \
        cudaError_t e = (x);                                                                   \
        if (e != cudaSuccess) {                                                                \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__);     \
            exit(2);                                                                           \
        }                                                                                      \
    } while (0)

static float bf(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

struct Rng {
    std::mt19937 g;
    explicit Rng(unsigned s) : g(s) {}
    float normal(float sd = 1.f) {
        std::normal_distribution<float> d(0.f, sd);
        return d(g);
    }
};

static std::vector<__nv_bfloat16> to_bf16(const std::vector<float>& v) {
    std::vector<__nv_bfloat16> o(v.size());
    for (size_t i = 0; i < v.size(); ++i) o[i] = __float2bfloat16_rn(v[i]);
    return o;
}
template <class T>
static T* dev_copy(const std::vector<T>& h) {
    T* d;
    CK(cudaMalloc(&d, h.size() * sizeof(T) + 16));
    CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
}

static int g_fail = 0;

static bool report(const char* name, double max_err, double max_ref, double tol, long long bad) {
    const bool ok = bad == 0 && std::isfinite(max_err);
    printf("[%s] %-58s max_abs_err=%.4g max_ref=%.4g tol=%.3g bad=%lld\n", ok ? "PASS" : "FAIL", name, max_err, max_ref,
           tol, bad);
    if (!ok) g_fail++;
    fflush(stdout);
    return ok;
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
static bool test_gemm(int M, int N, int K, int act, bool with_bias, bool with_res, bool with_rowvec, int sample,
                      bool identity = false, bool verbose_fail = false) {
    Rng rng(1234 + M * 7 + N * 3 + K);
    std::vector<float> A((size_t)M * K), W((size_t)N * K), bias(N), res, rowvec;
    for (auto& v : A) v = bf(rng.normal());
    for (auto& v : W) v = bf(rng.normal(1.0f / sqrtf((float)K)));
    if (identity) {
        for (int n = 0; n < N; ++n)
            for (int k = 0; k < K; ++k) W[(size_t)n * K + k] = (n == k) ? 1.f : 0.f;
    }
    for (auto& v : bias) v = with_bias ? bf(rng.normal(0.5f)) : 0.f;
    const int n_out = act == 2 ? N / 2 : N;
    const int rows_per_batch = with_rowvec ? (M + 1) / 2 : 0;
    if (with_res) {
        res.resize((size_t)M * n_out);
        for (auto& v : res) v = bf(rng.normal());
    }
    if (with_rowvec) {
        rowvec.resize((size_t)2 * N);
        for (auto& v : rowvec) v = rng.normal(0.5f);
    }
    auto Ab = to_bf16(A), Wb = to_bf16(W);
    __nv_bfloat16 *dA = dev_copy(Ab), *dW = dev_copy(Wb), *dOut, *dRes = nullptr;
    float *dBias = dev_copy(bias), *dRow = nullptr;
    CK(cudaMalloc(&dOut, (size_t)M * n_out * 2 + 16));
    CK(cudaMemset(dOut, 0xFF, (size_t)M * n_out * 2));
    if (with_res) {
        auto rb = to_bf16(res);
        dRes = dev_copy(rb);
    }
    if (with_rowvec) dRow = dev_copy(rowvec);
    supir_epilogue ep{};
    ep.bias = with_bias ? dBias : nullptr;
    ep.rowvec = dRow;
    ep.rows_per_batch = rows_per_batch;
    ep.rowvec_ld = N;
    ep.residual = dRes;
    ep.ldr = n_out;
    ep.act = act;
    int rc = supir_gemm_bf16(dA, K, dW, K, dOut, n_out, M, N, K, &ep, nullptr);
    if (rc) {
        printf("supir_gemm_bf16 rc=%d: %s\n", rc, supir_last_error());
        g_fail++;
        return false;
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("kernel failed: %s\n", cudaGetErrorString(e));
        exit(3);
    }
    std::vector<__nv_bfloat16> out((size_t)M * n_out);
    CK(cudaMemcpy(out.data(), dOut, out.size() * 2, cudaMemcpyDeviceToHost));
    // reference on sampled entries
    double max_err = 0, max_ref = 0;
    long long bad = 0;
    std::mt19937 pick(99);
    const long long total = (long long)M * n_out;
    const long long checks = sample > 0 && sample < total ? sample : total;
    int printed = 0;
    for (long long t = 0; t < checks; ++t) {
        long long idx = (checks == total) ? t : (long long)(pick() % total);
        const int m = (int)(idx / n_out), o = (int)(idx % n_out);
        auto acc_col = [&](int n) {
            double s = 0;
            for (int k = 0; k < K; ++k) s += (double)A[(size_t)m * K + k] * W[(size_t)n * K + k];
            s += bias[n];
            if (with_rowvec) s += rowvec[(size_t)(m / rows_per_batch) * N + n];
            return (float)s;
        };
        float ref;
        if (act == 2) {
            const int g = o / 16, j = o % 16;
            const float xv = bf(acc_col(g * 32 + j)), gv = bf(acc_col(g * 32 + 16 + j));
            ref = bf(xv * bf(0.5f * gv * (1.f + erff(gv * 0.70710678f))));
        } else {
            ref = bf(acc_col(o));
            if (act == 1) ref = ref / (1.f + expf(-ref));
        }
        if (with_res) ref += res[(size_t)m * n_out + o];
        const float got = __bfloat162float(out[(size_t)m * n_out + o]);
        const double err = fabs((double)got - ref);
        const double tol = 0.02 + 0.02 * fabs(ref);
        if (!(err <= tol)) {
            bad++;
            if (verbose_fail && printed < 12) {
                printf("   mismatch m=%d o=%d got=%g ref=%g\n", m, o, got, ref);
                printed++;
            }
        }
        if (err > max_err || !std::isfinite(err)) max_err = err;
        if (fabs(ref) > max_ref) max_ref = fabs(ref);
    }
    char name[256];
    snprintf(name, sizeof(name), "gemm M=%d N=%d K=%d act=%d bias=%d res=%d rowvec=%d%s", M, N, K, act, with_bias,
             with_res, with_rowvec, identity ? " identity" : "");
    bool ok = report(name, max_err, max_ref, 0.02, bad);
    cudaFree(dA); cudaFree(dW); cudaFree(dOut); cudaFree(dBias);
    if (dRes) cudaFree(dRes);
    if (dRow) cudaFree(dRow);
    return ok;
}

// ------------------------------------------------------------------------------------------------
// conv3x3
// ------------------------------------------------------------------------------------------------
static bool test_conv(int B, int H, int Wd, int Cin, int Cout, int sample, bool with_res, bool with_rowvec) {
    Rng rng(77 + H * 5 + Wd + Cin + Cout);
    std::vector<float> X((size_t)B * H * Wd * Cin), Wt((size_t)Cout * 9 * Cin), bias(Cout), res, rowvec;
    for (auto& v : X) v = bf(rng.normal());
    for (auto& v : Wt) v = bf(rng.normal(1.0f / sqrtf(9.f * Cin)));
    for (auto& v : bias) v = bf(rng.normal(0.5f));
    if (with_res) {
        res.resize((size_t)B * H * Wd * Cout);
        for (auto& v : res) v = bf(rng.normal());
    }
    if (with_rowvec) {
        rowvec.resize((size_t)B * Cout);
        for (auto& v : rowvec) v = rng.normal(0.5f);
    }
    auto Xb = to_bf16(X), Wb = to_bf16(Wt);
    __nv_bfloat16 *dX = dev_copy(Xb), *dW = dev_copy(Wb), *dOut, *dRes = nullptr;
    float *dBias = dev_copy(bias), *dRow = nullptr;
    const size_t on = (size_t)B * H * Wd * Cout;
    CK(cudaMalloc(&dOut, on * 2 + 16));
    CK(cudaMemset(dOut, 0xFF, on * 2));
    if (with_res) {
        auto rb = to_bf16(res);
        dRes = dev_copy(rb);
    }
    if (with_rowvec) dRow = dev_copy(rowvec);
    supir_epilogue ep{};
    ep.bias = dBias;
    ep.rowvec = dRow;
    ep.rowvec_ld = Cout;
    ep.residual = dRes;
    ep.ldr = Cout;
    int rc = supir_conv3x3_bf16(dX, Cin, dW, dOut, Cout, B, H, Wd, Cin, Cout, &ep, nullptr);
    if (rc) {
        printf("supir_conv3x3_bf16 rc=%d: %s\n", rc, supir_last_error());
        g_fail++;
        return false;
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("kernel failed: %s\n", cudaGetErrorString(e));
        exit(3);
    }
    std::vector<__nv_bfloat16> out(on);
    CK(cudaMemcpy(out.data(), dOut, on * 2, cudaMemcpyDeviceToHost));
    double max_err = 0, max_ref = 0;
    long long bad = 0;
    std::mt19937 pick(5);
    const long long total = (long long)on;
    const long long checks = sample > 0 && sample < total ? sample : total;
    for (long long t = 0; t < checks; ++t) {
        long long idx = (checks == total) ? t : (long long)(pick() % total);
        const int co = (int)(idx % Cout);
        long long pix = idx / Cout;
        const int x = (int)(pix % Wd);
        const int y = (int)((pix / Wd) % H);
        const int b = (int)(pix / ((long long)Wd * H));
        double s = bias[co];
        for (int dy = 0; dy < 3; ++dy)
            for (int dx = 0; dx < 3; ++dx) {
                const int yy = y + dy - 1, xx = x + dx - 1;
                if (yy < 0 || yy >= H || xx < 0 || xx >= Wd) continue;
                const float* xp = &X[(((size_t)b * H + yy) * Wd + xx) * Cin];
                const float* wp = &Wt[((size_t)co * 9 + dy * 3 + dx) * Cin];
                for (int c = 0; c < Cin; ++c) s += (double)xp[c] * wp[c];
            }
        if (with_rowvec) s += rowvec[(size_t)b * Cout + co];
        float ref = bf((float)s);
        if (with_res) ref += res[idx];
        const float got = __bfloat162float(out[idx]);
        const double err = fabs((double)got - ref);
        if (!(err <= 0.02 + 0.02 * fabs(ref))) bad++;
        if (err > max_err || !std::isfinite(err)) max_err = err;
        if (fabs(ref) > max_ref) max_ref = fabs(ref);
    }
    char name[256];
    snprintf(name, sizeof(name), "conv3x3 B=%d H=%d W=%d Cin=%d Cout=%d res=%d rowvec=%d", B, H, Wd, Cin, Cout, with_res,
             with_rowvec);
    bool ok = report(name, max_err, max_ref, 0.02, bad);
    cudaFree(dX); cudaFree(dW); cudaFree(dOut); cudaFree(dBias);
    if (dRes) cudaFree(dRes);
    if (dRow) cudaFree(dRow);
    return ok;
}

// ------------------------------------------------------------------------------------------------
// perf
// ------------------------------------------------------------------------------------------------
static void perf_gemm(int M, int N, int K, int act, int bn) {
    __nv_bfloat16 *dA, *dW, *dOut;
    CK(cudaMalloc(&dA, (size_t)M * K * 2));
    CK(cudaMalloc(&dW, (size_t)N * K * 2));
    CK(cudaMalloc(&dOut, (size_t)M * N * 2));
    CK(cudaMemset(dA, 0x11, (size_t)M * K * 2));
    CK(cudaMemset(dW, 0x11, (size_t)N * K * 2));
    supir_epilogue ep{};
    ep.act = act;
    supir_set_gemm_tile_n(bn);
    const int n_out = act == 2 ? N / 2 : N;
    for (int i = 0; i < 3; ++i) supir_gemm_bf16(dA, K, dW, K, dOut, n_out, M, N, K, &ep, nullptr);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20;
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) supir_gemm_bf16(dA, K, dW, K, dOut, n_out, M, N, K, &ep, nullptr);
    cudaEventRecord(e1);
    CK(cudaEventSynchronize(e1));
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    ms /= iters;
    printf("[PERF] gemm M=%d N=%d K=%d act=%d bn=%d : %.3f ms  %.1f TFLOP/s\n", M, N, K, act, bn, ms,
           2.0 * M * N * K / ms / 1e9);
    supir_set_gemm_tile_n(0);
    cudaFree(dA); cudaFree(dW); cudaFree(dOut);
    fflush(stdout);
}

// pseudo-random bf16 fill (hash of the index, roughly uniform in [-amp, amp]): realistic operand toggling for power / timing
__global__ void fill_random_bf16(__nv_bfloat16* p, size_t n, float amp, uint32_t seed) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t h = (uint32_t)i * 2654435761u ^ seed;
        h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
        p[i] = __float2bfloat16_rn(((h >> 8) * (1.0f / 8388608.0f) - 1.0f) * amp);
    }
}

static void perf_conv(int B, int H, int Wd, int Cin, int Cout, int bn) {
    __nv_bfloat16 *dX, *dW, *dOut;
    CK(cudaMalloc(&dX, (size_t)B * H * Wd * Cin * 2));
    CK(cudaMalloc(&dW, (size_t)Cout * 9 * Cin * 2));
    CK(cudaMalloc(&dOut, (size_t)B * H * Wd * Cout * 2));
    CK(cudaMemset(dX, 0x11, (size_t)B * H * Wd * Cin * 2));
    CK(cudaMemset(dW, 0x11, (size_t)Cout * 9 * Cin * 2));
    supir_set_gemm_tile_n(bn);
    for (int i = 0; i < 3; ++i) supir_conv3x3_bf16(dX, Cin, dW, dOut, Cout, B, H, Wd, Cin, Cout, nullptr, nullptr);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20;
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) supir_conv3x3_bf16(dX, Cin, dW, dOut, Cout, B, H, Wd, Cin, Cout, nullptr, nullptr);
    cudaEventRecord(e1);
    CK(cudaEventSynchronize(e1));
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    ms /= iters;
    printf("[PERF] conv3x3 B=%d H=%d W=%d Cin=%d Cout=%d bn=%d : %.3f ms  %.1f TFLOP/s\n", B, H, Wd, Cin, Cout, bn, ms,
           2.0 * B * H * Wd * Cout * 9.0 * Cin / ms / 1e9);
    supir_set_gemm_tile_n(0);
    cudaFree(dX); cudaFree(dW); cudaFree(dOut);
    fflush(stdout);
}


// ------------------------------------------------------------------------------------------------
// attention
// ------------------------------------------------------------------------------------------------
static bool test_attention(int B, int H, int Lq, int Lk, int sample_rows) {
    Rng rng(4242 + Lq + Lk * 3 + H);
    const int C = H * 64;
    std::vector<float> Q((size_t)B * Lq * C), K((size_t)B * Lk * C), V((size_t)B * Lk * C);
    for (auto& v : Q) v = bf(rng.normal(1.5f));
    for (auto& v : K) v = bf(rng.normal(1.5f));
    for (auto& v : V) v = bf(rng.normal());
    auto Qb = to_bf16(Q), Kb = to_bf16(K), Vb = to_bf16(V);
    __nv_bfloat16 *dQ = dev_copy(Qb), *dK = dev_copy(Kb), *dV = dev_copy(Vb), *dO;
    CK(cudaMalloc(&dO, (size_t)B * Lq * C * 2 + 16));
    CK(cudaMemset(dO, 0xFF, (size_t)B * Lq * C * 2));
    const float scale = 0.125f;
    int rc = supir_attention_bf16(dQ, C, dK, C, dV, C, dO, C, B, H, Lq, Lk, 64, scale, nullptr);
    if (rc) {
        printf("supir_attention_bf16 rc=%d: %s\n", rc, supir_last_error());
        g_fail++;
        return false;
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("attention kernel failed: %s\n", cudaGetErrorString(e));
        exit(3);
    }
    std::vector<__nv_bfloat16> out((size_t)B * Lq * C);
    CK(cudaMemcpy(out.data(), dO, out.size() * 2, cudaMemcpyDeviceToHost));
    double max_err = 0, max_ref = 0;
    long long bad = 0;
    std::mt19937 pick(17);
    const long long rows_total = (long long)B * H * Lq;
    const long long checks = sample_rows > 0 && sample_rows < rows_total ? sample_rows : rows_total;
    std::vector<double> sc(Lk);
    for (long long t = 0; t < checks; ++t) {
        const long long idx = checks == rows_total ? t : (long long)(pick() % rows_total);
        const int i = (int)(idx % Lq);
        const int h = (int)((idx / Lq) % H);
        const int b = (int)(idx / ((long long)Lq * H));
        const float* q = &Q[((size_t)b * Lq + i) * C + h * 64];
        double mx = -1e30;
        for (int j = 0; j < Lk; ++j) {
            const float* k = &K[((size_t)b * Lk + j) * C + h * 64];
            double s = 0;
            for (int d = 0; d < 64; ++d) s += (double)q[d] * k[d];
            sc[j] = s * scale;
            if (sc[j] > mx) mx = sc[j];
        }
        double den = 0;
        for (int j = 0; j < Lk; ++j) { sc[j] = exp(sc[j] - mx); den += sc[j]; }
        for (int d = 0; d < 64; ++d) {
            double o = 0;
            for (int j = 0; j < Lk; ++j) o += sc[j] * V[((size_t)b * Lk + j) * C + h * 64 + d];
            const float ref = (float)(o / den);
            const float got = __bfloat162float(out[((size_t)b * Lq + i) * C + h * 64 + d]);
            const double err = fabs((double)got - ref);
            if (!(err <= 0.02 + 0.02 * fabs(ref))) bad++;
            if (err > max_err || !std::isfinite(err)) max_err = err;
            if (fabs(ref) > max_ref) max_ref = fabs(ref);
        }
    }
    char name[256];
    snprintf(name, sizeof(name), "attention B=%d H=%d Lq=%d Lk=%d", B, H, Lq, Lk);
    bool ok = report(name, max_err, max_ref, 0.02, bad);
    cudaFree(dQ); cudaFree(dK); cudaFree(dV); cudaFree(dO);
    return ok;
}

static void perf_attention(int B, int H, int Lq, int Lk) {
    const int C = H * 64;
    __nv_bfloat16 *dQ, *dK, *dV, *dO;
    CK(cudaMalloc(&dQ, (size_t)B * Lq * C * 2));
    CK(cudaMalloc(&dK, (size_t)B * Lk * C * 2));
    CK(cudaMalloc(&dV, (size_t)B * Lk * C * 2));
    CK(cudaMalloc(&dO, (size_t)B * Lq * C * 2));
    fill_random_bf16<<<1024, 256>>>(dQ, (size_t)B * Lq * C, 2.0f, 1u);
    fill_random_bf16<<<1024, 256>>>(dK, (size_t)B * Lk * C, 2.0f, 2u);
    fill_random_bf16<<<1024, 256>>>(dV, (size_t)B * Lk * C, 1.0f, 3u);
    for (int i = 0; i < 3; ++i) supir_attention_bf16(dQ, C, dK, C, dV, C, dO, C, B, H, Lq, Lk, 64, 0.125f, nullptr);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 10;
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) supir_attention_bf16(dQ, C, dK, C, dV, C, dO, C, B, H, Lq, Lk, 64, 0.125f, nullptr);
    cudaEventRecord(e1);
    CK(cudaEventSynchronize(e1));
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    ms /= iters;
    printf("[PERF] attention B=%d H=%d Lq=%d Lk=%d : %.3f ms  %.1f TFLOP/s\n", B, H, Lq, Lk, ms,
           4.0 * B * H * (double)Lq * Lk * 64 / ms / 1e9);
    cudaFree(dQ); cudaFree(dK); cudaFree(dV); cudaFree(dO);
    fflush(stdout);
}


// data / bias / duration sensitivity of the GEMM (power cap, epilogue cost): constant vs random operands, with/without bias+residual
static void perf_gemm_variants(int M, int N, int K, int act) {
    const int n_out = act == 2 ? N / 2 : N;
    Rng rng(5);
    std::vector<float> hA((size_t)M * K), hW((size_t)N * K), hb(N);
    for (auto& v : hA) v = rng.normal();
    for (auto& v : hW) v = rng.normal(1.0f / sqrtf((float)K));
    for (auto& v : hb) v = rng.normal(0.3f);
    auto Ab = to_bf16(hA), Wb = to_bf16(hW);
    __nv_bfloat16 *dA = dev_copy(Ab), *dW = dev_copy(Wb), *dOut, *dRes, *cA, *cW;
    float* dB = dev_copy(hb);
    CK(cudaMalloc(&dOut, (size_t)M * n_out * 2));
    CK(cudaMalloc(&dRes, (size_t)M * n_out * 2));
    CK(cudaMemset(dRes, 0x3c, (size_t)M * n_out * 2));
    CK(cudaMalloc(&cA, (size_t)M * K * 2));
    CK(cudaMalloc(&cW, (size_t)N * K * 2));
    CK(cudaMemset(cA, 0x11, (size_t)M * K * 2));
    CK(cudaMemset(cW, 0x11, (size_t)N * K * 2));
    struct V { const char* name; bool rnd, bias, res; int iters; } vs[] = {
        {"const data, no bias", false, false, false, 20}, {"random data, no bias", true, false, false, 20},
        {"random data, bias", true, true, false, 20},     {"random data, bias+res", true, true, true, 20},
        {"random data, bias, 300 iters", true, true, false, 300}};
    for (auto& v : vs) {
        supir_epilogue ep{};
        ep.act = act;
        ep.bias = v.bias ? dB : nullptr;
        ep.residual = v.res ? dRes : nullptr;
        ep.ldr = n_out;
        const __nv_bfloat16 *a = v.rnd ? dA : cA, *w = v.rnd ? dW : cW;
        for (int i = 0; i < 3; ++i) supir_gemm_bf16(a, K, w, K, dOut, n_out, M, N, K, &ep, nullptr);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0);
        for (int i = 0; i < v.iters; ++i) supir_gemm_bf16(a, K, w, K, dOut, n_out, M, N, K, &ep, nullptr);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        ms /= v.iters;
        printf("[PERF3] gemm M=%d N=%d K=%d act=%d %-32s: %.3f ms  %.1f TFLOP/s\n", M, N, K, act, v.name, ms, 2.0 * M * N * K / ms / 1e9);
        fflush(stdout);
    }
    cudaFree(dA); cudaFree(dW); cudaFree(dOut); cudaFree(dRes); cudaFree(cA); cudaFree(cW); cudaFree(dB);
}

int main(int argc, char** argv) {
    std::string what = argc > 1 ? argv[1] : "all";
    int dev = 0;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    printf("device: %s sm_%d%d SMs=%d\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
    if (what == "gemm" || what == "all") {
        for (int bn : {64, 128, 160, 256}) {
            supir_set_gemm_tile_n(bn);
            test_gemm(128, 256, 64, 0, false, false, false, 0);
            test_gemm(128, 256, 256, 0, true, false, false, 0);
            test_gemm(300, 200, 192, 0, true, true, false, 0);
            test_gemm(1000, 328, 320, 1, true, false, true, 0);
        }
        supir_set_gemm_tile_n(0);
        test_gemm(2, 1280, 320, 0, true, false, false, 0);
        test_gemm(154, 640, 2048, 0, false, false, false, 20000);
        test_gemm(2048, 1280, 1280, 0, true, true, false, 20000);
        test_gemm(8192, 5120, 640, 2, true, false, false, 20000);
        test_gemm(2048, 2560, 1280, 2, true, true, false, 20000);
        test_gemm(20000, 640, 640, 0, true, true, false, 20000);  // > 132 tiles: the persistent tile loop wraps
    }
    if (what == "conv" || what == "all") {
        test_conv(1, 16, 16, 64, 64, 0, false, false);
        test_conv(2, 32, 32, 64, 128, 0, true, true);
        test_conv(1, 17, 23, 72, 40, 0, false, false);
        test_conv(2, 64, 64, 320, 320, 20000, true, true);
        test_conv(2, 32, 32, 2560, 1280, 5000, false, true);
        test_conv(1, 150, 150, 128, 128, 20000, false, false);
        test_conv(2, 8, 8, 128, 256, 0, false, false);
    }
    if (what == "attnpack") {   // bf16 packing of the probabilities on the ALU pipe (0..4 of 4 pairs) instead of the XU-pipe conversion
        for (int n : {0, 2, 3, 4}) {
            printf("-- %d of 4 pairs packed with integer instructions\n", n);
            supir_set_attention_alu_pack(n);
            perf_attention(98, 10, 4096, 4096);
            perf_attention(98, 20, 1024, 1024);
            perf_attention(98, 20, 1024, 77);
        }
        for (int n : {2, 4}) {
            supir_set_attention_alu_pack(n);
            test_attention(2, 10, 1024, 1024, 500);
            test_attention(1, 2, 333, 500, 0);
            test_attention(2, 3, 200, 77, 0);
        }
        supir_set_attention_alu_pack(-1);
    }
    if (what == "attnquick") {     // hang guard for a GPU session: every kernel variant once, small
        for (int emu : {0, 2}) {
            supir_set_attention_exp_emulation(emu);
            test_attention(1, 2, 128, 256, 0);
            test_attention(2, 3, 200, 77, 0);
            test_attention(1, 2, 333, 128, 0);
            test_attention(1, 2, 333, 500, 0);
            test_attention(40, 8, 512, 512, 200);     // 1280 CTAs: several waves over the SMs
            test_attention(60, 8, 256, 77, 200);
        }
        supir_set_attention_exp_emulation(-1);
    }
    if (what == "attn" || what == "all") {
      for (int emu : {0, 2}) {
        printf("-- softmax exponent emulation %d of 4 pairs\n", emu);
        supir_set_attention_exp_emulation(emu);
        test_attention(1, 1, 128, 128, 0);
        test_attention(1, 2, 128, 256, 0);
        test_attention(2, 3, 200, 77, 0);
        test_attention(1, 2, 333, 500, 0);
        test_attention(2, 10, 1024, 1024, 2000);
        test_attention(2, 20, 4096, 4096, 500);
        test_attention(2, 10, 4096, 77, 2000);
        test_attention(3, 2, 700, 96, 0);
        test_attention(3, 2, 300, 128, 0);
        test_attention(40, 20, 1024, 1024, 300);      // many more CTAs than SMs: several waves
      }
      supir_set_attention_exp_emulation(-1);
    }
    if (what == "attnperf" || what == "all") {
        perf_attention(2, 10, 4096, 4096);
        perf_attention(2, 20, 1024, 1024);
        perf_attention(2, 10, 16384, 16384);
        perf_attention(2, 10, 4096, 77);
        perf_attention(2, 20, 1024, 77);
    }
    if (what == "attnperf2") {   // the shapes of the 49-window step (batch 98), for every exponent-emulation setting
        for (int emu : {0, 2}) {
            printf("-- softmax exponent emulation %d of 4 pairs\n", emu);
            supir_set_attention_exp_emulation(emu);
            perf_attention(98, 10, 4096, 4096);
            perf_attention(98, 20, 1024, 1024);
            perf_attention(98, 10, 4096, 77);
            perf_attention(98, 20, 1024, 77);
        }
        supir_set_attention_exp_emulation(-1);
    }
    if (what == "sanitize") {   // small cases for compute-sanitizer (memcheck / racecheck / synccheck)
        for (int bn : {0, 64, 160}) {
            supir_set_gemm_tile_n(bn);
            test_gemm(300, 200, 192, 0, true, true, false, 0);
            test_gemm(130, 328, 320, 1, true, false, true, 0);
            test_gemm(200, 256, 128, 2, true, false, false, 0);
        }
        supir_set_gemm_tile_n(0);
        test_conv(2, 32, 32, 64, 128, 0, true, true);
        test_conv(1, 17, 23, 72, 40, 0, false, false);
        test_attention(2, 3, 200, 77, 0);
        test_attention(1, 2, 333, 500, 0);
    }
    if (what == "perf3" || what == "all") {
        perf_gemm_variants(14336, 10240, 1280, 2);
        perf_gemm_variants(14336, 1280, 1280, 0);
        perf_gemm_variants(57344, 640, 640, 0);
        perf_gemm_variants(57344, 5120, 640, 2);
        perf_gemm_variants(8192, 8192, 8192, 0);
    }
    if (what == "perf2" || what == "all") {
        // shapes of the tiled workload at 8 windows per launch (B = 16): calibrates the tile-width cost model
        struct Sh { int M, N, K, act; } shapes[] = {
            {16384, 1280, 1280, 0}, {16384, 3840, 1280, 0}, {16384, 10240, 1280, 2}, {16384, 1280, 5120, 0},
            {65536, 640, 640, 0}, {65536, 1920, 640, 0}, {65536, 5120, 640, 2}, {65536, 640, 2560, 0},
            {2048, 1280, 1280, 0}, {2048, 3840, 1280, 0}, {8192, 640, 640, 0}, {1232, 163840, 2048, 0}};
        for (auto& sh : shapes)
            for (int bn : {0, 128, 160, 256}) perf_gemm(sh.M, sh.N, sh.K, sh.act, bn);
        for (int bn : {0, 128, 160, 256}) {
            perf_conv(16, 32, 32, 1280, 1280, bn);
            perf_conv(16, 64, 64, 640, 640, bn);
            perf_conv(16, 128, 128, 320, 320, bn);
            perf_conv(16, 32, 32, 2560, 1280, bn);
            perf_conv(16, 128, 128, 128, 1280, bn);
        }
    }
    if (what == "perf" || what == "all") {
        for (int bn : {128, 256}) {
            perf_gemm(8192, 1280, 1280, 0, bn);
            perf_gemm(8192, 10240, 1280, 2, bn);
            perf_gemm(8192, 1280, 5120, 0, bn);
            perf_gemm(32768, 640, 640, 0, bn);
            perf_gemm(2048, 1280, 1280, 0, bn);
            perf_gemm(8192, 8192, 8192, 0, bn);
            perf_conv(2, 128, 128, 320, 320, bn);
            perf_conv(2, 32, 32, 1280, 1280, bn);
            perf_conv(8, 32, 32, 1280, 1280, bn);
            perf_conv(2, 64, 64, 640, 640, bn);
        }
    }
    printf("== selftest done: %d failure(s)\n", g_fail);
    return g_fail ? 1 : 0;
}
