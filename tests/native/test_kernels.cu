// SPDX-License-Identifier: Apache-2.0
// Stand-alone bring-up harness for libhcpb200 (no Python, no torch): checks the wgmma GEMM / conv kernels
// against naive CUDA-core reference kernels on the same GPU and prints achieved TFLOP/s.  Test infrastructure
// only -- the parity tests proper live in tests/test_*.py and go through the same C ABI.
//
//   build: see Makefile in this directory;   run on an H100:  timeout 600 tests/native/test_kernels [filter]
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <vector>
#include <string>
#include "../../include/hcp_b200.h"

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);     \
            exit(2);                                                                            \
        }                                                                                       \
    } while (0)

static int g_fail = 0, g_pass = 0;
static const char* g_filter = nullptr;
static bool want(const char* name) { return !g_filter || strstr(name, g_filter); }

// ------------------------------------------------------------------------------------------
__global__ void fill_bf16(__nv_bfloat16* p, size_t n, uint32_t seed, float scale) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u + seed * 0x9E3779B9u;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    float f = ((x & 0xFFFFFF) / 16777216.0f) * 2.f - 1.f;
    p[i] = __float2bfloat16(f * scale);
}
__global__ void fill_f32(float* p, size_t n, uint32_t seed, float scale) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u + seed * 0x9E3779B9u;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    p[i] = (((x & 0xFFFFFF) / 16777216.0f) * 2.f - 1.f) * scale;
}
static __nv_bfloat16* alloc_bf16(size_t n, uint32_t seed, float scale = 1.f) {
    __nv_bfloat16* p;
    CK(cudaMalloc(&p, n * 2 + 256));
    fill_bf16<<<(unsigned)((n + 255) / 256), 256>>>(p, n, seed, scale);
    return p;
}
static float* alloc_f32(size_t n, uint32_t seed, float scale = 1.f) {
    float* p;
    CK(cudaMalloc(&p, n * 4 + 256));
    fill_f32<<<(unsigned)((n + 255) / 256), 256>>>(p, n, seed, scale);
    return p;
}

// out = sum_s A_s B_s^T (+bias +rowbias +residual), fp32 accumulate, fp32 result
struct RefSeg { const __nv_bfloat16* a; const __nv_bfloat16* b; int64_t lda, ldb, k, nrb; };
__global__ void gemm_ref(RefSeg s0, RefSeg s1, RefSeg s2, int nseg, int64_t M, int64_t N, const float* bias,
                         const float* rowbias, int64_t rpg, const __nv_bfloat16* res, int64_t ldr, float* out) {
    int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t m = blockIdx.y;
    if (n >= N || m >= M) return;
    RefSeg segs[3] = {s0, s1, s2};
    float acc = 0.f;
    for (int s = 0; s < nseg; ++s) {
        if (n >= segs[s].nrb) continue;
        for (int64_t k = 0; k < segs[s].k; ++k)
            acc += __bfloat162float(segs[s].a[m * segs[s].lda + k]) * __bfloat162float(segs[s].b[n * segs[s].ldb + k]);
    }
    if (bias) acc += bias[n];
    if (rowbias) acc += rowbias[(m / rpg) * N + n];
    if (res) acc += __bfloat162float(res[m * ldr + n]);
    out[m * N + n] = acc;
}

// mode 0: conv stride s pad 1.  mode 1: transposed (dgrad of stride 2) with w[co][kh][kw][ci] = dgrad arrangement
__global__ void conv_ref(const __nv_bfloat16* x, const __nv_bfloat16* w, int B, int Hin, int Win, int Cin, int Cout,
                         int stride, int mode, const float* bias, const float* rowbias, const __nv_bfloat16* res,
                         float* out) {
    const int Ho = mode == 0 ? Hin / stride : Hin * 2, Wo = mode == 0 ? Win / stride : Win * 2;
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t total = (int64_t)B * Ho * Wo * Cout;
    if (idx >= total) return;
    int co = idx % Cout;
    int64_t pix = idx / Cout;
    int wo = pix % Wo, ho = (pix / Wo) % Ho, b = pix / ((int64_t)Wo * Ho);
    float acc = 0.f;
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            int ih, iw;
            if (mode == 0) { ih = ho * stride + kh - 1; iw = wo * stride + kw - 1; }
            else {
                int th = ho + 1 - kh, tw = wo + 1 - kw;
                if ((th & 1) || (tw & 1)) continue;
                ih = th / 2; iw = tw / 2;
                if (th < 0 || tw < 0) continue;
            }
            if (ih < 0 || iw < 0 || ih >= Hin || iw >= Win) continue;
            const __nv_bfloat16* xp = x + (((int64_t)b * Hin + ih) * Win + iw) * Cin;
            const __nv_bfloat16* wp = w + ((int64_t)co * 9 + kh * 3 + kw) * Cin;
            for (int c = 0; c < Cin; ++c) acc += __bfloat162float(xp[c]) * __bfloat162float(wp[c]);
        }
    if (bias) acc += bias[co];
    if (rowbias) acc += rowbias[(int64_t)b * Cout + co];
    if (res) acc += __bfloat162float(res[idx]);
    out[idx] = acc;
}

__global__ void cmp_kernel(const __nv_bfloat16* got, int64_t ldg, const float* ref, int64_t M, int64_t N,
                           double* stats /* sum_err2, sum_ref2, max_abs_err, max_abs_ref */) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= M * N) return;
    int64_t m = i / N, n = i % N;
    float g = __bfloat162float(got[m * ldg + n]);
    float r = ref[i];
    float e = fabsf(g - r);
    atomicAdd(&stats[0], (double)e * e);
    atomicAdd(&stats[1], (double)r * r);
    // max via atomicMax on the bit pattern of non-negative doubles
    atomicMax((unsigned long long*)&stats[2], (unsigned long long)__double_as_longlong((double)e));
    atomicMax((unsigned long long*)&stats[3], (unsigned long long)__double_as_longlong((double)fabsf(r)));
    if (isnan(g)) atomicAdd(&stats[4], 1.0);
}

static bool compare(const char* name, const __nv_bfloat16* got, int64_t ldg, const float* ref, int64_t M, int64_t N,
                    double tol_rel = 6e-3) {
    double* d;
    CK(cudaMalloc(&d, 5 * sizeof(double)));
    CK(cudaMemset(d, 0, 5 * sizeof(double)));
    cmp_kernel<<<(unsigned)((M * N + 255) / 256), 256>>>(got, ldg, ref, M, N, d);
    double h[5];
    CK(cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost));
    CK(cudaFree(d));
    double rel = sqrt(h[0] / (h[1] + 1e-30));
    bool ok = rel < tol_rel && h[4] == 0 && h[1] > 0;
    printf("[%s] %-58s relL2=%.3e maxerr=%.3e maxref=%.3e nan=%g\n", ok ? "PASS" : "FAIL", name, rel, h[2], h[3], h[4]);
    fflush(stdout);
    if (ok) ++g_pass; else ++g_fail;
    return ok;
}

static float time_ms(void (*fn)(void*), void* ctx, int iters) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) fn(ctx);
    CK(cudaEventRecord(e0));
    for (int i = 0; i < iters; ++i) fn(ctx);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    return ms / iters;
}

// ------------------------------------------------------------------------------------------
struct GemmCase {
    const char* name; int64_t M, N, K0; int64_t K1; int64_t r1;  // second segment: K1 = padded (64), r1 valid rows-cols
    bool bias, rowbias, res; bool timeit;
};
static void run_gemm_case(const GemmCase& c) {
    if (!want(c.name)) return;
    hcp_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.nseg = c.K1 > 0 ? 2 : 1;
    __nv_bfloat16* A0 = alloc_bf16(c.M * c.K0, 1, 1.f);
    __nv_bfloat16* B0 = alloc_bf16(c.N * c.K0, 2, 1.f / sqrtf((float)c.K0));
    __nv_bfloat16 *A1 = nullptr, *B1 = nullptr;
    a.a[0] = A0; a.b[0] = B0; a.lda[0] = c.K0; a.ldb[0] = c.K0; a.k[0] = c.K0; a.n_rows_b[0] = c.N;
    if (c.K1 > 0) {
        A1 = alloc_bf16(c.M * c.K1, 3, 1.f);     // [M, 64] with garbage beyond r1: only r1 columns are declared
        B1 = alloc_bf16(c.N * c.K1, 4, 0.3f);
        a.a[1] = A1; a.b[1] = B1; a.lda[1] = c.K1; a.ldb[1] = c.K1; a.k[1] = c.r1; a.n_rows_b[1] = c.N;
    }
    a.M = c.M; a.N = c.N;
    float* bias = c.bias ? alloc_f32(c.N, 5, 0.5f) : nullptr;
    const int64_t rpg = 64;
    float* rowbias = c.rowbias ? alloc_f32(((c.M + rpg - 1) / rpg) * c.N, 6, 0.5f) : nullptr;
    __nv_bfloat16* res = c.res ? alloc_bf16(c.M * c.N, 7, 1.f) : nullptr;
    a.bias = bias; a.rowbias = rowbias; a.rows_per_group = rpg; a.residual = res; a.ldr = c.N;
    __nv_bfloat16* out;
    CK(cudaMalloc(&out, c.M * c.N * 2));
    CK(cudaMemset(out, 0xFF, c.M * c.N * 2));
    a.out = out; a.ldo = c.N;
    int rc = hcp_gemm_bf16(&a, 0);
    if (rc) { printf("[FAIL] %s: hcp_gemm_bf16 rc=%d %s\n", c.name, rc, hcp_last_error_string()); ++g_fail; return; }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("[FAIL] %s: kernel error %s\n", c.name, cudaGetErrorString(e)); ++g_fail; exit(3); }
    float* ref;
    CK(cudaMalloc(&ref, c.M * c.N * 4));
    RefSeg s0{A0, B0, c.K0, c.K0, c.K0, c.N}, s1{A1, B1, c.K1, c.K1, c.r1, c.N}, s2{};
    gemm_ref<<<dim3((unsigned)((c.N + 127) / 128), (unsigned)c.M), 128>>>(s0, s1, s2, a.nseg, c.M, c.N, bias, rowbias, rpg, res, c.N, ref);
    compare(c.name, out, c.N, ref, c.M, c.N);
    if (c.timeit) {
        struct Ctx { hcp_gemm_args* a; } ctx{&a};
        float ms = time_ms([](void* p) { hcp_gemm_bf16(((Ctx*)p)->a, 0); }, &ctx, 20);
        double fl = 2.0 * c.M * c.N * (c.K0 + c.r1);
        printf("       %-58s %.3f ms  %.1f TFLOP/s\n", c.name, ms, fl / ms * 1e-9);
    }
    cudaFree(A0); cudaFree(B0); if (A1) cudaFree(A1); if (B1) cudaFree(B1);
    if (bias) cudaFree(bias); if (rowbias) cudaFree(rowbias); if (res) cudaFree(res);
    cudaFree(out); cudaFree(ref);
}

struct ConvCase { const char* name; int B, H, W, Cin, Cout, stride, mode; bool bias, rowbias, res, timeit; };
static void run_conv_case(const ConvCase& c) {
    if (!want(c.name)) return;
    const int Ho = c.mode == 0 ? c.H / c.stride : c.H * 2, Wo = c.mode == 0 ? c.W / c.stride : c.W * 2;
    size_t nx = (size_t)c.B * c.H * c.W * c.Cin, nw = (size_t)c.Cout * 9 * c.Cin, no = (size_t)c.B * Ho * Wo * c.Cout;
    __nv_bfloat16* x = alloc_bf16(nx, 11, 1.f);
    __nv_bfloat16* w = alloc_bf16(nw, 12, 1.f / sqrtf(9.f * c.Cin));
    float* bias = c.bias ? alloc_f32(c.Cout, 13, 0.5f) : nullptr;
    float* rowbias = c.rowbias ? alloc_f32((size_t)c.B * c.Cout, 14, 0.5f) : nullptr;
    __nv_bfloat16* res = c.res ? alloc_bf16(no, 15, 1.f) : nullptr;
    __nv_bfloat16* out;
    CK(cudaMalloc(&out, no * 2));
    CK(cudaMemset(out, 0xFF, no * 2));
    hcp_conv3x3_args a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.w = w; a.B = c.B; a.Hin = c.H; a.Win = c.W; a.Cin = c.Cin; a.Cout = c.Cout; a.stride = c.stride; a.mode = c.mode;
    a.bias = bias; a.rowbias = rowbias; a.residual = res; a.out = out;
    int rc = hcp_conv3x3_bf16(&a, 0);
    if (rc) { printf("[FAIL] %s: hcp_conv3x3_bf16 rc=%d %s\n", c.name, rc, hcp_last_error_string()); ++g_fail; return; }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("[FAIL] %s: kernel error %s\n", c.name, cudaGetErrorString(e)); ++g_fail; exit(3); }
    float* ref;
    CK(cudaMalloc(&ref, no * 4));
    conv_ref<<<(unsigned)((no + 255) / 256), 256>>>(x, w, c.B, c.H, c.W, c.Cin, c.Cout, c.stride, c.mode, bias, rowbias, res, ref);
    compare(c.name, out, c.Cout, ref, (int64_t)c.B * Ho * Wo, c.Cout);
    if (c.timeit) {
        struct Ctx { hcp_conv3x3_args* a; } ctx{&a};
        float ms = time_ms([](void* p) { hcp_conv3x3_bf16(((Ctx*)p)->a, 0); }, &ctx, 10);
        double fl = 2.0 * c.B * Ho * Wo * (double)c.Cout * 9 * c.Cin * (c.mode == 1 ? 0.25 : 1.0);
        printf("       %-58s %.3f ms  %.1f TFLOP/s\n", c.name, ms, fl / ms * 1e-9);
    }
    cudaFree(x); cudaFree(w); if (bias) cudaFree(bias); if (rowbias) cudaFree(rowbias); if (res) cudaFree(res);
    cudaFree(out); cudaFree(ref);
}

void run_attn_tests(const char* filter, int* pass, int* fail);    // test_attn.cu (optional, weak)
__attribute__((weak)) void run_attn_tests(const char*, int*, int*) {}

int main(int argc, char** argv) {
    if (argc > 1) g_filter = argv[1];
    int rc = hcp_device_check();
    printf("hcp_version=%d device_check=%d (%s)\n", hcp_version(), rc, hcp_last_error_string());
    if (rc) return 2;

    // smallest first: a dead-lock or descriptor error shows up on the cheapest case
    const GemmCase gemm_cases[] = {
        {"gemm 128x64x64", 128, 64, 64, 0, 0, false, false, false, false},
        {"gemm 128x32x128 (BN=32)", 128, 32, 128, 0, 0, false, false, false, false},
        {"gemm 128x128x256", 128, 128, 256, 0, 0, false, false, false, false},
        {"gemm 256x320x320 (BN=160)", 256, 320, 320, 0, 0, false, false, false, false},
        {"gemm 200x320x320 ragged M +bias", 200, 320, 320, 0, 0, true, false, false, false},
        {"gemm 64x1280x1280 +bias+res", 64, 1280, 1280, 0, 0, true, false, true, false},
        {"gemm 1024x640x640 +lora r8 +bias+res", 1024, 640, 640, 64, 8, true, false, true, false},
        {"gemm 1024x960x320 +lora r24 (qkv)", 1024, 960, 320, 64, 24, false, false, false, false},
        {"gemm 512x320x768 +rowbias (cross kv K=768)", 512, 320, 768, 0, 0, false, true, false, false},
        {"gemm 77x640x768 ragged", 77, 640, 768, 0, 0, false, false, false, false},
        {"gemm 16384x24x320 (lora down, N=24)", 16384, 24, 320, 0, 0, false, false, false, true},
        {"gemm 16384x320x320 +lora r8 +bias+res", 16384, 320, 320, 64, 8, true, false, true, true},
        {"gemm 16384x2560x320 (ff proj)", 16384, 2560, 320, 0, 0, true, false, false, true},
        {"gemm 16384x320x1280 (ff out)", 16384, 320, 1280, 0, 0, true, false, true, true},
        {"gemm 4096x5120x640", 4096, 5120, 640, 0, 0, true, false, false, true},
        {"gemm 8192x8192x8192 (peak probe)", 8192, 8192, 8192, 0, 0, false, false, false, true},
    };
    for (const auto& c : gemm_cases) run_gemm_case(c);

    const ConvCase conv_cases[] = {
        {"conv s1 B1 16x16 64->64", 1, 16, 16, 64, 64, 1, 0, false, false, false, false},
        {"conv s1 B2 8x8 128->64 (2 img/tile)", 2, 8, 8, 128, 64, 1, 0, true, false, false, false},
        {"conv s1 B3 8x8 64->320 (ragged img)", 3, 8, 8, 64, 320, 1, 0, true, true, true, false},
        {"conv s1 B2 32x32 320->320 +bias+rowbias+res", 2, 32, 32, 320, 320, 1, 0, true, true, true, false},
        {"conv s1 B1 64x64 320->320", 1, 64, 64, 320, 320, 1, 0, true, true, false, false},
        {"conv s2 B2 32x32 320->320", 2, 32, 32, 320, 320, 2, 0, true, false, false, false},
        {"conv s2 B2 16x16 64->128", 2, 16, 16, 64, 128, 2, 0, false, false, false, false},
        {"conv s2 B4 64x64 320->320", 4, 64, 64, 320, 320, 2, 0, true, false, false, true},
        {"conv dgrad-s2 B2 8x8 128->64", 2, 8, 8, 128, 64, 2, 1, false, false, false, false},
        {"conv dgrad-s2 B2 16x16 320->320", 2, 16, 16, 320, 320, 2, 1, false, false, false, false},
        {"conv dgrad-s2 B4 32x32 320->320", 4, 32, 32, 320, 320, 2, 1, false, false, false, true},
        {"conv s1 B4 64x64 320->320 (timed)", 4, 64, 64, 320, 320, 1, 0, true, true, false, true},
        {"conv s1 B4 64x64 960->320 (timed)", 4, 64, 64, 960, 320, 1, 0, true, true, false, true},
        {"conv s1 B4 32x32 640->640 (timed)", 4, 32, 32, 640, 640, 1, 0, true, true, false, true},
        {"conv s1 B4 16x16 1280->1280 (timed)", 4, 16, 16, 1280, 1280, 1, 0, true, true, false, true},
        {"conv s1 B4 8x8 2560->1280 (timed)", 4, 8, 8, 2560, 1280, 1, 0, true, true, false, true},
    };
    for (const auto& c : conv_cases) run_conv_case(c);

    run_attn_tests(g_filter, &g_pass, &g_fail);

    printf("SUMMARY pass=%d fail=%d\n", g_pass, g_fail);
    return g_fail ? 1 : 0;
}
