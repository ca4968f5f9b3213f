// Standalone micro-benchmark for fe_mul variants (throughput on independent chains + equality with the portable path).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I distaff_b200/csrc -o /tmp/bench_modmul tools/bench_modmul.cu && /tmp/bench_modmul
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "fp128.cuh"
using namespace dg;

#define DG_HAVE_V3 1
template <int V> __device__ __forceinline__ fe mulv(fe a, fe b) {
#ifdef __CUDA_ARCH__
    if (V == 1) return ptx::fe_mul_v1(a, b);
    if (V == 2) return ptx::fe_mul_v3(a, b);
    if (V == 3) return ptx::fe_mul_v4(a, b);
    if (V == 4) return ptx::fe_mul_v4t<false>(a, b);      // the NTT pass kernels' multiply: rare canonicalisation inline, no call
#endif
    return portable::fe_mul(a, b);
}

template <int V>
__global__ void __launch_bounds__(256) tput(const fe *in, fe *out, int iters) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    fe x0 = in[i], x1 = in[i + 1], x2 = in[i + 2], x3 = in[i + 3], m = in[i + 4];
    for (int k = 0; k < iters; k++) { x0 = mulv<V>(x0, m); x1 = mulv<V>(x1, m); x2 = mulv<V>(x2, m); x3 = mulv<V>(x3, m); }
    out[i] = fe_add(fe_add(x0, x1), fe_add(x2, x3));
}
// butterfly-like mix: add, sub, mul
template <int V>
__global__ void __launch_bounds__(256) tput_bfly(const fe *in, fe *out, int iters) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    fe a = in[i], b = in[i + 1], c = in[i + 2], d = in[i + 3], w = in[i + 4];
    for (int k = 0; k < iters; k++) {
        fe s = fe_add(a, b), t = mulv<V>(fe_sub(a, b), w); a = s; b = t;
        fe s2 = fe_add(c, d), t2 = mulv<V>(fe_sub(c, d), w); c = s2; d = t2;
    }
    out[i] = fe_add(fe_add(a, b), fe_add(c, d));
}
// ---- call-structure experiment at the occupancy of the real kernels (16 warps/SM): 4 independent butterflies per iteration with
//      (0) inlined multiplies, (1) one out-of-line multiply per butterfly, (2) one out-of-line call per PAIR of multiplies
struct fe2 { fe a, b; };
#ifdef __CUDA_ARCH__
static __device__ __noinline__ fe mul1_call(fe a, fe b) { return ptx::fe_mul_v4t<false>(a, b); }
static __device__ __noinline__ fe2 mul2_call(fe a0, fe b0, fe a1, fe b1) { fe2 r; r.a = ptx::fe_mul_v4t<false>(a0, b0); r.b = ptx::fe_mul_v4t<false>(a1, b1); return r; }
#endif
template <int MODE>
__global__ void __launch_bounds__(256, 2) tput_call(const fe *in, fe *out, int iters) {
    extern __shared__ unsigned char pad[];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    fe x[8], w = in[i + 8];
#pragma unroll
    for (int q = 0; q < 8; q++) x[q] = in[i + q];
    if (iters < 0) pad[threadIdx.x] = 1;
#ifdef __CUDA_ARCH__
    for (int k = 0; k < iters; k++) {
        fe d[4];
#pragma unroll
        for (int q = 0; q < 4; q++) { fe a = x[2 * q], b = x[2 * q + 1]; x[2 * q] = fe_add(a, b); d[q] = fe_sub(a, b); }
        if (MODE == 0) {
#pragma unroll
            for (int q = 0; q < 4; q++) x[2 * q + 1] = ptx::fe_mul_v4(d[q], w);
        } else if (MODE == 1) {
#pragma unroll
            for (int q = 0; q < 4; q++) x[2 * q + 1] = mul1_call(d[q], w);
        } else {
#pragma unroll
            for (int q = 0; q < 4; q += 2) { fe2 r = mul2_call(d[q], w, d[q + 1], w); x[2 * q + 1] = r.a; x[2 * q + 3] = r.b; }
        }
        // rotate so that the chains mix
        fe t = x[1]; x[1] = x[3]; x[3] = x[5]; x[5] = x[7]; x[7] = t;
    }
#endif
    fe s = x[0];
#pragma unroll
    for (int q = 1; q < 8; q++) s = fe_add(s, x[q]);
    out[i] = s;
}
template <int MODE> void run_call(const char *name, fe *d_in, fe *d_out, int blocks, int iters) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaFuncSetAttribute(tput_call<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    float best = 1e9;
    for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(e0);
        tput_call<MODE><<<blocks, 256, 100 * 1024>>>(d_in, d_out, iters);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    printf("%-22s %8.3f ms  %7.1f Gbfly/s (16 warps/SM)\n", name, best, (double)blocks * 256 * iters * 4 / best / 1e6);
}

template <int V> __global__ void check(const fe *a, const fe *b, fe *o, int n) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) o[i] = mulv<V>(a[i], b[i]); }

template <int V> void run(const char *name, fe *d_in, fe *d_out, int blocks, int iters) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int kind = 0; kind < 2; kind++) {
        float best = 1e9;
        for (int rep = 0; rep < 3; rep++) {
            cudaEventRecord(e0);
            if (kind == 0) tput<V><<<blocks, 256>>>(d_in, d_out, iters); else tput_bfly<V><<<blocks, 256>>>(d_in, d_out, iters);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
        }
        double ops = (double)blocks * 256 * iters * (kind == 0 ? 4 : 2);
        printf("%-10s %-6s %8.3f ms  %7.1f G%s/s\n", name, kind == 0 ? "mul" : "bfly", best, ops / best / 1e6, kind == 0 ? "mul" : "bfly");
    }
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int blocks = sms * 8, iters = 2000, n = blocks * 256 + 16;
    std::vector<fe> h(n);
    unsigned long long s = 88172645463325252ULL;
    auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
    for (auto &x : h) { x.lo = rnd(); x.hi = rnd(); if (x.hi == ~0ULL) x.hi = 12345; }
    // edge cases at the front
    const fe edge[] = {{0, 0}, {1, 0}, {DG_M_LO - 1, DG_M_HI}, {DG_M_LO - 2, DG_M_HI}, {~0ULL, 0}, {0, 1}, {0, 1ULL << 63}, {DG_C_LO, 0}, {DG_C_LO + 1, 0}, {0xffffffffULL, 0xffffffff00000000ULL}};
    const int ne = sizeof(edge) / sizeof(edge[0]);
    std::vector<fe> ea, eb;
    for (int i = 0; i < ne; i++) for (int j = 0; j < ne; j++) { ea.push_back(edge[i]); eb.push_back(edge[j]); }
    for (int i = 0; i < 200000; i++) { ea.push_back(h[i % n]); eb.push_back(h[(i * 7 + 3) % n]); }
    {   // crafted pairs (tools/gen_mul_vectors.py): products whose partially reduced value overflows 2^128 / has an all-ones top limb
        FILE *f = fopen("tools/_bin/mul_vectors.bin", "rb");
        if (f) { fe ab[2]; int cnt = 0; while (fread(ab, 16, 2, f) == 2) { ea.push_back(ab[0]); eb.push_back(ab[1]); cnt++; } fclose(f); printf("%d crafted pairs\n", cnt); }
        else printf("tools/_bin/mul_vectors.bin not found: crafted pairs skipped\n");
    }
    fe *d_in, *d_out, *da, *db, *d0, *d1;
    cudaMalloc(&d_in, n * 16); cudaMalloc(&d_out, n * 16);
    cudaMemcpy(d_in, h.data(), n * 16, cudaMemcpyHostToDevice);
    int m = ea.size();
    cudaMalloc(&da, m * 16); cudaMalloc(&db, m * 16); cudaMalloc(&d0, m * 16); cudaMalloc(&d1, m * 16);
    cudaMemcpy(da, ea.data(), m * 16, cudaMemcpyHostToDevice); cudaMemcpy(db, eb.data(), m * 16, cudaMemcpyHostToDevice);
    std::vector<fe> r0(m), r1(m);
    check<0><<<(m + 255) / 256, 256>>>(da, db, d0, m); cudaMemcpy(r0.data(), d0, m * 16, cudaMemcpyDeviceToHost);
    auto cmp = [&](const char *nm) { cudaMemcpy(r1.data(), d1, m * 16, cudaMemcpyDeviceToHost); int bad = 0; for (int i = 0; i < m; i++) if (r0[i].lo != r1[i].lo || r0[i].hi != r1[i].hi) { if (bad < 3) printf("  %s mismatch at %d\n", nm, i); bad++; } printf("%s vs portable: %d mismatches of %d\n", nm, bad, m); };
    check<1><<<(m + 255) / 256, 256>>>(da, db, d1, m); cmp("ptx");
#ifdef DG_HAVE_V3
    check<2><<<(m + 255) / 256, 256>>>(da, db, d1, m); cmp("v3");
#endif
    check<3><<<(m + 255) / 256, 256>>>(da, db, d1, m); cmp("v4");
    check<4><<<(m + 255) / 256, 256>>>(da, db, d1, m); cmp("v4 inline");
    run<0>("portable", d_in, d_out, blocks, iters);
    run<1>("ptx", d_in, d_out, blocks, iters);
#ifdef DG_HAVE_V3
    run<2>("v3", d_in, d_out, blocks, iters);
#endif
    run<3>("v4", d_in, d_out, blocks, iters);
    run<4>("v4 inline", d_in, d_out, blocks, iters);
    run_call<0>("bfly inline", d_in, d_out, blocks, iters / 2);
    run_call<1>("bfly 1 mul per call", d_in, d_out, blocks, iters / 2);
    run_call<2>("bfly 2 muls per call", d_in, d_out, blocks, iters / 2);
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
