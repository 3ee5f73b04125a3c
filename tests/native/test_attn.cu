// SPDX-License-Identifier: Apache-2.0
// Attention fwd/bwd bring-up tests (test infrastructure): wgmma kernels vs naive fp32 CUDA-core references.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include "../../include/hcp_b200.h"

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);     \
            exit(2);                                                                            \
        }                                                                                       \
    } while (0)

__global__ void afill_bf16(__nv_bfloat16* p, size_t n, uint32_t seed, float scale) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u + seed * 0x9E3779B9u;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    p[i] = __float2bfloat16((((x & 0xFFFFFF) / 16777216.0f) * 2.f - 1.f) * scale);
}
__global__ void afill_f32(float* p, size_t n, uint32_t seed, float scale, float offset) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u + seed * 0x9E3779B9u;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    p[i] = (((x & 0xFFFFFF) / 16777216.0f) * 2.f - 1.f) * scale + offset;
}

struct AP {
    const __nv_bfloat16 *q, *k, *v, *dout;
    int64_t ldq, ldk, ldv, lddo;
    int B, H, Lq, Lkv, d;
    float scale;
    const float* bias;
};

// one thread per (b,h,q): O row (fp32), lse
__global__ void attn_ref_fwd(AP a, float* O /*[B,Lq,H*d]*/, float* lse /*[B,H,Lq]*/) {
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= (int64_t)a.B * a.H * a.Lq) return;
    int q = idx % a.Lq, h = (idx / a.Lq) % a.H, b = idx / ((int64_t)a.Lq * a.H);
    const __nv_bfloat16* qp = a.q + ((int64_t)b * a.Lq + q) * a.ldq + h * a.d;
    float m = -INFINITY;
    for (int j = 0; j < a.Lkv; ++j) {
        const __nv_bfloat16* kp = a.k + ((int64_t)b * a.Lkv + j) * a.ldk + h * a.d;
        float s = 0;
        for (int e = 0; e < a.d; ++e) s += __bfloat162float(qp[e]) * __bfloat162float(kp[e]);
        s = s * a.scale + (a.bias ? a.bias[(int64_t)b * a.Lkv + j] : 0.f);
        m = fmaxf(m, s);
    }
    float l = 0;
    float acc[192];
    for (int e = 0; e < a.d; ++e) acc[e] = 0;
    for (int j = 0; j < a.Lkv; ++j) {
        const __nv_bfloat16* kp = a.k + ((int64_t)b * a.Lkv + j) * a.ldk + h * a.d;
        const __nv_bfloat16* vp = a.v + ((int64_t)b * a.Lkv + j) * a.ldv + h * a.d;
        float s = 0;
        for (int e = 0; e < a.d; ++e) s += __bfloat162float(qp[e]) * __bfloat162float(kp[e]);
        s = s * a.scale + (a.bias ? a.bias[(int64_t)b * a.Lkv + j] : 0.f);
        float p = expf(s - m);
        l += p;
        for (int e = 0; e < a.d; ++e) acc[e] += p * __bfloat162float(vp[e]);
    }
    float* op = O + ((int64_t)b * a.Lq + q) * (a.H * a.d) + h * a.d;
    for (int e = 0; e < a.d; ++e) op[e] = acc[e] / l;
    lse[idx] = m + logf(l);   // idx == (b*H + h)*Lq + q
}

// one thread per (b,h,q): dQ row; uses O (fp32 ref) for delta
__global__ void attn_ref_dq(AP a, const float* O, const float* lse, float* dQ) {
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= (int64_t)a.B * a.H * a.Lq) return;
    int q = idx % a.Lq, h = (idx / a.Lq) % a.H, b = idx / ((int64_t)a.Lq * a.H);
    const __nv_bfloat16* qp = a.q + ((int64_t)b * a.Lq + q) * a.ldq + h * a.d;
    const __nv_bfloat16* gp = a.dout + ((int64_t)b * a.Lq + q) * a.lddo + h * a.d;
    const float* op = O + ((int64_t)b * a.Lq + q) * (a.H * a.d) + h * a.d;
    float delta = 0;
    for (int e = 0; e < a.d; ++e) delta += __bfloat162float(gp[e]) * op[e];
    float acc[192];
    for (int e = 0; e < a.d; ++e) acc[e] = 0;
    for (int j = 0; j < a.Lkv; ++j) {
        const __nv_bfloat16* kp = a.k + ((int64_t)b * a.Lkv + j) * a.ldk + h * a.d;
        const __nv_bfloat16* vp = a.v + ((int64_t)b * a.Lkv + j) * a.ldv + h * a.d;
        float s = 0, dp = 0;
        for (int e = 0; e < a.d; ++e) {
            s += __bfloat162float(qp[e]) * __bfloat162float(kp[e]);
            dp += __bfloat162float(gp[e]) * __bfloat162float(vp[e]);
        }
        s = s * a.scale + (a.bias ? a.bias[(int64_t)b * a.Lkv + j] : 0.f);
        float p = expf(s - lse[idx]);
        float ds = p * (dp - delta) * a.scale;
        for (int e = 0; e < a.d; ++e) acc[e] += ds * __bfloat162float(kp[e]);
    }
    float* dq = dQ + ((int64_t)b * a.Lq + q) * (a.H * a.d) + h * a.d;
    for (int e = 0; e < a.d; ++e) dq[e] = acc[e];
}

// one thread per (b,h,kv): dK, dV rows
__global__ void attn_ref_dkv(AP a, const float* O, const float* lse, float* dK, float* dV) {
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= (int64_t)a.B * a.H * a.Lkv) return;
    int j = idx % a.Lkv, h = (idx / a.Lkv) % a.H, b = idx / ((int64_t)a.Lkv * a.H);
    const __nv_bfloat16* kp = a.k + ((int64_t)b * a.Lkv + j) * a.ldk + h * a.d;
    const __nv_bfloat16* vp = a.v + ((int64_t)b * a.Lkv + j) * a.ldv + h * a.d;
    float ak[192], av[192];
    for (int e = 0; e < a.d; ++e) ak[e] = av[e] = 0;
    const float bj = a.bias ? a.bias[(int64_t)b * a.Lkv + j] : 0.f;
    for (int q = 0; q < a.Lq; ++q) {
        const __nv_bfloat16* qp = a.q + ((int64_t)b * a.Lq + q) * a.ldq + h * a.d;
        const __nv_bfloat16* gp = a.dout + ((int64_t)b * a.Lq + q) * a.lddo + h * a.d;
        const float* op = O + ((int64_t)b * a.Lq + q) * (a.H * a.d) + h * a.d;
        float s = 0, dp = 0, delta = 0;
        for (int e = 0; e < a.d; ++e) {
            s += __bfloat162float(qp[e]) * __bfloat162float(kp[e]);
            dp += __bfloat162float(gp[e]) * __bfloat162float(vp[e]);
            delta += __bfloat162float(gp[e]) * op[e];
        }
        s = s * a.scale + bj;
        float p = expf(s - lse[((int64_t)b * a.H + h) * a.Lq + q]);
        float ds = p * (dp - delta) * a.scale;
        for (int e = 0; e < a.d; ++e) {
            av[e] += p * __bfloat162float(gp[e]);
            ak[e] += ds * __bfloat162float(qp[e]);
        }
    }
    float* dk = dK + ((int64_t)b * a.Lkv + j) * (a.H * a.d) + h * a.d;
    float* dv = dV + ((int64_t)b * a.Lkv + j) * (a.H * a.d) + h * a.d;
    for (int e = 0; e < a.d; ++e) { dk[e] = ak[e]; dv[e] = av[e]; }
}

__global__ void acmp_kernel(const __nv_bfloat16* got, int64_t ldg, const float* ref, int64_t M, int64_t N, double* st) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= M * N) return;
    int64_t m = i / N, n = i % N;
    float g = __bfloat162float(got[m * ldg + n]), r = ref[i];
    float e = fabsf(g - r);
    atomicAdd(&st[0], (double)e * e);
    atomicAdd(&st[1], (double)r * r);
    if (isnan(g) || isinf(g)) atomicAdd(&st[2], 1.0);
}
static bool acompare(const char* name, const char* what, const __nv_bfloat16* got, int64_t ldg, const float* ref, int64_t M,
                     int64_t N, double tol, int* pass, int* fail) {
    double* d;
    CK(cudaMalloc(&d, 3 * sizeof(double)));
    CK(cudaMemset(d, 0, 3 * sizeof(double)));
    acmp_kernel<<<(unsigned)((M * N + 255) / 256), 256>>>(got, ldg, ref, M, N, d);
    double h[3];
    CK(cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost));
    CK(cudaFree(d));
    double rel = sqrt(h[0] / (h[1] + 1e-30));
    bool ok = rel < tol && h[2] == 0 && h[1] > 0;
    printf("[%s] %-44s %-3s relL2=%.3e nan=%g\n", ok ? "PASS" : "FAIL", name, what, rel, h[2]);
    fflush(stdout);
    if (ok) ++*pass; else ++*fail;
    return ok;
}

struct AttnCase { const char* name; int B, H, Lq, Lkv, d; bool self_fused; bool bias; bool check; bool timeit; bool bwd; };

static void run_attn_case(const AttnCase& c, int* pass, int* fail) {
    const int C = c.H * c.d;
    // self_fused: q,k,v live in one [B, L, 3C] buffer (as the fused QKV projection writes them)
    const int64_t ldq = c.self_fused ? 3 * C : C, ldkv = c.self_fused ? 3 * C : 2 * C;
    __nv_bfloat16 *qbuf, *kvbuf = nullptr;
    const float amp = 1.5f;
    size_t nq = (size_t)c.B * c.Lq * ldq, nkv = (size_t)c.B * c.Lkv * ldkv;
    CK(cudaMalloc(&qbuf, nq * 2));
    afill_bf16<<<(unsigned)((nq + 255) / 256), 256>>>(qbuf, nq, 21, amp);
    const __nv_bfloat16 *q = qbuf, *k, *v;
    if (c.self_fused) { k = qbuf + C; v = qbuf + 2 * C; }
    else {
        CK(cudaMalloc(&kvbuf, nkv * 2));
        afill_bf16<<<(unsigned)((nkv + 255) / 256), 256>>>(kvbuf, nkv, 22, amp);
        k = kvbuf; v = kvbuf + C;
    }
    size_t no = (size_t)c.B * c.Lq * C, nko = (size_t)c.B * c.Lkv * C;
    __nv_bfloat16 *o, *dout, *dq, *dk, *dv;
    CK(cudaMalloc(&o, no * 2)); CK(cudaMalloc(&dout, no * 2)); CK(cudaMalloc(&dq, no * 2));
    CK(cudaMalloc(&dk, nko * 2)); CK(cudaMalloc(&dv, nko * 2));
    CK(cudaMemset(o, 0xFF, no * 2)); CK(cudaMemset(dq, 0xFF, no * 2)); CK(cudaMemset(dk, 0xFF, nko * 2)); CK(cudaMemset(dv, 0xFF, nko * 2));
    afill_bf16<<<(unsigned)((no + 255) / 256), 256>>>(dout, no, 23, 1.0f);
    float *lse, *bias = nullptr, *ws;
    CK(cudaMalloc(&lse, (size_t)c.B * c.H * c.Lq * 4));
    if (c.bias) {
        CK(cudaMalloc(&bias, (size_t)c.B * c.Lkv * 4));
        afill_f32<<<(unsigned)((c.B * c.Lkv + 255) / 256), 256>>>(bias, (size_t)c.B * c.Lkv, 24, 2.0f, 0.f);
    }
    size_t wsb = hcp_attn_bwd_workspace_bytes(c.B, c.H, c.Lq, c.Lkv, c.d);
    CK(cudaMalloc(&ws, wsb));
    const float scale = 1.f / sqrtf((float)c.d);

    hcp_attn_args fa;
    memset(&fa, 0, sizeof(fa));
    fa.q = q; fa.ldq = ldq; fa.k = k; fa.ldk = ldkv; fa.v = v; fa.ldv = ldkv;
    fa.B = c.B; fa.H = c.H; fa.Lq = c.Lq; fa.Lkv = c.Lkv; fa.d = c.d; fa.scale = scale; fa.kv_bias = bias;
    fa.o = o; fa.ldo = C; fa.lse = lse;
    int rc = hcp_attn_fwd_bf16(&fa, 0);
    if (rc) { printf("[FAIL] %s fwd rc=%d %s\n", c.name, rc, hcp_last_error_string()); ++*fail; return; }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("[FAIL] %s: fwd kernel error %s\n", c.name, cudaGetErrorString(e)); ++*fail; exit(3); }

    hcp_attn_bwd_args ba;
    memset(&ba, 0, sizeof(ba));
    ba.q = q; ba.ldq = ldq; ba.k = k; ba.ldk = ldkv; ba.v = v; ba.ldv = ldkv; ba.o = o; ba.ldo = C; ba.dout = dout; ba.lddo = C;
    ba.B = c.B; ba.H = c.H; ba.Lq = c.Lq; ba.Lkv = c.Lkv; ba.d = c.d; ba.scale = scale; ba.kv_bias = bias; ba.lse = lse;
    ba.dq = dq; ba.lddq = C; ba.dk = dk; ba.lddk = C; ba.dv = dv; ba.lddv = C; ba.workspace = ws; ba.workspace_bytes = wsb;
    if (c.bwd) {
        rc = hcp_attn_bwd_bf16(&ba, 0);
        if (rc) { printf("[FAIL] %s bwd rc=%d %s\n", c.name, rc, hcp_last_error_string()); ++*fail; return; }
        e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("[FAIL] %s: bwd kernel error %s\n", c.name, cudaGetErrorString(e)); ++*fail; exit(3); }
    }
    if (c.check) {
        AP a{q, k, v, dout, ldq, ldkv, ldkv, C, c.B, c.H, c.Lq, c.Lkv, c.d, scale, bias};
        float *rO, *rlse, *rdQ, *rdK, *rdV;
        CK(cudaMalloc(&rO, no * 4)); CK(cudaMalloc(&rlse, (size_t)c.B * c.H * c.Lq * 4));
        CK(cudaMalloc(&rdQ, no * 4)); CK(cudaMalloc(&rdK, nko * 4)); CK(cudaMalloc(&rdV, nko * 4));
        int64_t nt = (int64_t)c.B * c.H * c.Lq;
        attn_ref_fwd<<<(unsigned)((nt + 63) / 64), 64>>>(a, rO, rlse);
        acompare(c.name, "O", o, C, rO, (int64_t)c.B * c.Lq, C, 1.5e-2, pass, fail);
        if (c.bwd) {
            attn_ref_dq<<<(unsigned)((nt + 63) / 64), 64>>>(a, rO, rlse, rdQ);
            int64_t nk = (int64_t)c.B * c.H * c.Lkv;
            attn_ref_dkv<<<(unsigned)((nk + 63) / 64), 64>>>(a, rO, rlse, rdK, rdV);
            acompare(c.name, "dQ", dq, C, rdQ, (int64_t)c.B * c.Lq, C, 2e-2, pass, fail);
            acompare(c.name, "dK", dk, C, rdK, (int64_t)c.B * c.Lkv, C, 2e-2, pass, fail);
            acompare(c.name, "dV", dv, C, rdV, (int64_t)c.B * c.Lkv, C, 2e-2, pass, fail);
        }
        cudaFree(rO); cudaFree(rlse); cudaFree(rdQ); cudaFree(rdK); cudaFree(rdV);
    }
    if (c.timeit) {
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        for (int i = 0; i < 2; ++i) hcp_attn_fwd_bf16(&fa, 0);
        CK(cudaEventRecord(e0));
        for (int i = 0; i < 10; ++i) hcp_attn_fwd_bf16(&fa, 0);
        CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= 10;
        double fl = 4.0 * c.B * c.H * (double)c.Lq * c.Lkv * c.d;
        printf("       %-44s fwd %.3f ms  %.1f TFLOP/s\n", c.name, ms, fl / ms * 1e-9);
        if (c.bwd) {
            for (int i = 0; i < 2; ++i) hcp_attn_bwd_bf16(&ba, 0);
            CK(cudaEventRecord(e0));
            for (int i = 0; i < 10; ++i) hcp_attn_bwd_bf16(&ba, 0);
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= 10;
            printf("       %-44s bwd %.3f ms  %.1f TFLOP/s (2x fwd flops convention: %.1f)\n", c.name, ms, 2.5 * fl / ms * 1e-9, 2.0 * fl / ms * 1e-9);
        }
    }
    cudaFree(qbuf); if (kvbuf) cudaFree(kvbuf); cudaFree(o); cudaFree(dout); cudaFree(dq); cudaFree(dk); cudaFree(dv);
    cudaFree(lse); if (bias) cudaFree(bias); cudaFree(ws);
}

void run_attn_tests(const char* filter, int* pass, int* fail) {
    const AttnCase cases[] = {
        {"attn B1 H2 L128 d64", 1, 2, 128, 128, 64, true, false, true, false, true},
        {"attn B2 H3 L256 d40", 2, 3, 256, 256, 40, true, false, true, false, true},
        {"attn B1 H2 Lq200 Lkv77 d40 cross", 1, 2, 200, 77, 40, false, false, true, false, true},
        {"attn B2 H2 Lq200 Lkv80 d40 cross +bias", 2, 2, 200, 80, 40, false, true, true, false, true},
        {"attn B2 H8 L1024 d80", 2, 8, 1024, 1024, 80, true, false, true, true, true},
        {"attn B2 H4 Lq1024 Lkv77 d80 cross", 2, 4, 1024, 77, 80, false, false, true, false, true},
        {"attn B2 H8 L256 d160", 2, 8, 256, 256, 160, true, false, true, false, true},
        {"attn B1 H8 L64 d160", 1, 8, 64, 64, 160, true, false, true, false, true},
        {"attn B2 H8 Lq64 Lkv77 d160 cross", 2, 8, 64, 77, 160, false, false, true, false, true},
        {"attn B1 H8 L4096 d40", 1, 8, 4096, 4096, 40, true, false, true, true, true},
        {"attn B4 H8 L4096 d40 (timed)", 4, 8, 4096, 4096, 40, true, false, false, true, true},
        {"attn B4 H8 Lq4096 Lkv77 d40 (timed)", 4, 8, 4096, 77, 40, false, false, false, true, true},
    };
    for (const auto& c : cases) {
        if (filter && !strstr(c.name, filter)) continue;
        run_attn_case(c, pass, fail);
    }
}
