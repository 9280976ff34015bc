// ubench_mix.cu -- stand-alone micro-benchmark / A-B check of the K1 slerp kernels (no torch, no liblb200).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo tools/ubench_mix.cu -o tools/ubench_mix
// V0   = round-1a register-resident cluster kernel (kept here only as the baseline and bit-exactness anchor:
//        it is the kernel the pytest parity suite validated against the torch oracle)
// S<T> = slerp_stage_kernel<__half, T, exact?> from latentblending_b200/csrc/mix_kernels.cuh
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../latentblending_b200/csrc/mix_kernels.cuh"

using namespace lbmix;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

namespace v0 {
constexpr int kThreads = 256;
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void block_reduce3(double& aa, double& bb, double& ab, double* sm /*[3*8]*/) {
    aa = warp_sum_d(aa);
    bb = warp_sum_d(bb);
    ab = warp_sum_d(ab);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) {
        sm[w] = aa;
        sm[8 + w] = bb;
        sm[16 + w] = ab;
    }
    __syncthreads();
    aa = bb = ab = 0.0;
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) {
        aa += sm[i];
        bb += sm[8 + i];
        ab += sm[16 + i];
    }
}

// ---- fast path: one cluster per row ----------------------------------------------
template <typename T, int CHUNKS>
__global__ void __launch_bounds__(kThreads)
slerp_cluster_kernel(const T* __restrict__ p0, const T* __restrict__ p1, T* __restrict__ out, int64_t n,
                     int64_t stride0, int64_t stride1, int64_t stride_out, double fract,
                     const double* __restrict__ fract_rows) {
    constexpr int VE = Vec<T>::N;
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned crank = cluster.block_rank();
    const unsigned csize = cluster.num_blocks();
    const int64_t row = blockIdx.y;
    const T* a_row = p0 + row * stride0;
    const T* b_row = p1 + row * stride1;
    T* o_row = out + row * stride_out;

    __shared__ double red[24];
    __shared__ double cta_sum[3];

    uint4 va[CHUNKS], vb[CHUNKS];
    int64_t off[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        int64_t v = ((int64_t)(crank * CHUNKS + c)) * kThreads + threadIdx.x;
        off[c] = v * VE;
        if (off[c] < n) {
            va[c] = ldg_stream(a_row + off[c]);
            vb[c] = ldg_stream(b_row + off[c]);
        } else {
            va[c] = make_uint4(0, 0, 0, 0);
            vb[c] = make_uint4(0, 0, 0, 0);
        }
    }
    double aa = 0.0, bb = 0.0, ab = 0.0;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        float fa[VE], fb[VE];
        Vec<T>::unpack(va[c], fa);
        Vec<T>::unpack(vb[c], fb);
#pragma unroll
        for (int e = 0; e < VE; ++e) {
            double da = fa[e], db = fb[e];
            aa = fma(da, da, aa);
            bb = fma(db, db, bb);
            ab = fma(da, db, ab);
        }
    }
    block_reduce3(aa, bb, ab, red);
    if (threadIdx.x == 0) {
        cta_sum[0] = aa;
        cta_sum[1] = bb;
        cta_sum[2] = ab;
    }
    cluster.sync();
    double taa = 0.0, tbb = 0.0, tab = 0.0;
    for (unsigned r = 0; r < csize; ++r) {
        const double* remote = cluster.map_shared_rank(cta_sum, r);
        taa += remote[0];
        tbb += remote[1];
        tab += remote[2];
    }
    cluster.sync();  // nobody may exit while a peer still reads its cta_sum
    const double f = fract_rows ? fract_rows[row] : fract;
    double s0, s1;
    slerp_weights(taa, tbb, tab, f, s0, s1);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        if (off[c] < n) {
            float fa[VE], fb[VE], fo[VE];
            Vec<T>::unpack(va[c], fa);
            Vec<T>::unpack(vb[c], fb);
#pragma unroll
            for (int e = 0; e < VE; ++e) fo[e] = slerp_elem(fa[e], fb[e], s0, s1);
            stg_stream(o_row + off[c], Vec<T>::pack(fo));
        }
    }
}


}  // namespace v0

// ---- inputs ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
__global__ void fill_normal(__half* p, size_t n, uint32_t seed, float scale) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t h1 = hash32((uint32_t)i * 2u + seed), h2 = hash32((uint32_t)i * 2u + 1u + seed * 31u);
        float u1 = (h1 + 1.0f) * (1.0f / 4294967296.0f), u2 = h2 * (1.0f / 4294967296.0f);
        p[i] = __float2half_rn(scale * sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2));
    }
}
// special rows: r%8: 0 normal, 1 tiny (fp16 subnormals), 2 huge, 3 b = a, 4 b = -a*(1+eps) (cancellation),
// 5 sparse zeros, 6 mixed magnitudes, 7 normal*0.01
__global__ void make_special(__half* a, __half* b, int rows, int n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)rows * n; i += (size_t)gridDim.x * blockDim.x) {
        int r = (int)(i / n);
        float x = __half2float(a[i]), y = __half2float(b[i]);
        switch (r & 7) {
            case 1: x *= 3e-6f; y *= 3e-6f; break;
            case 2: x *= 9000.f; y *= 9000.f; break;
            case 3: y = x; break;
            case 4: y = -x * 1.0009765625f; break;
            case 5: if (hash32((uint32_t)i) & 3) { x = 0.f; } if (hash32((uint32_t)i + 7u) & 1) { y = 0.f; } break;
            case 6: x *= exp2f((float)((int)(hash32((uint32_t)i) % 30) - 20)); y *= exp2f((float)((int)(hash32((uint32_t)i + 3u) % 30) - 20)); break;
            case 7: x *= 0.01f; y *= 0.01f; break;
            default: break;
        }
        a[i] = __float2half_rn(x);
        b[i] = __float2half_rn(y);
    }
}
__global__ void count_diff(const uint16_t* x, const uint16_t* y, size_t n, unsigned long long* cnt) {
    unsigned long long c = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) c += x[i] != y[i];
    if (c) atomicAdd(cnt, c);
}
// fraction of elements the certified path hands to the exact path (weights recomputed per row, one CTA per row)
__global__ void count_uncertified(const __half* p0, const __half* p1, int n, double fract, unsigned long long* cnt) {
    __shared__ double red[96];
    const __half* a = p0 + (size_t)blockIdx.x * n;
    const __half* b = p1 + (size_t)blockIdx.x * n;
    double aa = 0, bb = 0, ab = 0;
    for (int i = threadIdx.x; i < n; i += 256) {
        double x = __half2float(a[i]), y = __half2float(b[i]);
        aa += x * x; bb += y * y; ab += x * y;
    }
    block_reduce3<256>(aa, bb, ab, red);
    double s0, s1;
    slerp_weights(aa, bb, ab, fract, s0, s1);
    SplitW w(s0, s1);
    unsigned long long c = 0;
    for (int i = threadIdx.x; i < n; i += 256) {
        float E;
        float x = __half2float(a[i]), y = __half2float(b[i]);
        float r = slerp_fast(x, y, w, E);
        c += !slerp_certified(r, __half2float(__float2half_rn(r)), E);
    }
    if (c) atomicAdd(cnt, c);
}

// ---- launchers -----------------------------------------------------------------------------------
template <int CHUNKS>
void launch_v0(const __half* p0, const __half* p1, __half* out, int rows, int n, int csize, double f) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(csize, rows, 1);
    cfg.blockDim = dim3(256);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, v0::slerp_cluster_kernel<__half, CHUNKS>, p0, p1, out, (int64_t)n, (int64_t)n, (int64_t)n, (int64_t)n, f, (const double*)nullptr));
}
void run_v0(const __half* p0, const __half* p1, __half* out, int rows, int n, double f) {
    if (n == 65536) launch_v0<4>(p0, p1, out, rows, n, 8, f);
    else if (n == 16384) launch_v0<2>(p0, p1, out, rows, n, 4, f);
    else { printf("v0: unsupported n\n"); exit(1); }
}
template <int THREADS, bool EXACT>
void run_stage(const __half* p0, const __half* p1, __half* out, int rows, int n, int csize, double f) {
    auto kern = slerp_stage_kernel<__half, THREADS, EXACT>;
    int slice = ((n + csize - 1) / csize + 7) / 8 * 8;
    size_t smem = (size_t)slice * 4;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(csize, rows, 1);
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, kern, p0, p1, out, (int64_t)n, slice, (int64_t)n, (int64_t)n, (int64_t)n, f, (const double*)nullptr));
}

template <int THREADS, bool EXACT, bool HINT, int OCC = 1280>
void run_l2(const __half* p0, const __half* p1, __half* out, int rows, int n, int csize, double f) {
    auto kern = slerp_l2_kernel<__half, THREADS, EXACT, HINT, OCC>;
    int slice = ((n + csize - 1) / csize + 7) / 8 * 8;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(csize, rows, 1);
    cfg.blockDim = dim3(THREADS);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, kern, p0, p1, out, (int64_t)n, slice, (int64_t)n, (int64_t)n, (int64_t)n, f, (const double*)nullptr));
}

template <typename F> float time_ms(F f, int iters = 10, int warm = 3) {
    for (int i = 0; i < warm; ++i) f();
    CK(cudaDeviceSynchronize());
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    CK(cudaEventRecord(a));
    for (int i = 0; i < iters; ++i) f();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    return ms / iters;
}

int main(int argc, char** argv) {
    const double peak = argc > 1 ? atof(argv[1]) : 6573.5;   // measured HBM GB/s (MEASURED_PEAKS.json)
    const int maxrows = 2048, n = 65536;
    __half *p0, *p1, *o0, *o1;
    unsigned long long* cnt;
    size_t tot = (size_t)maxrows * n;
    CK(cudaMalloc(&p0, tot * 2)); CK(cudaMalloc(&p1, tot * 2)); CK(cudaMalloc(&o0, tot * 2)); CK(cudaMalloc(&o1, tot * 2));
    CK(cudaMalloc(&cnt, 8));
    fill_normal<<<1184, 256>>>(p0, tot, 1u, 1.0f);
    fill_normal<<<1184, 256>>>(p1, tot, 77u, 1.0f);
    make_special<<<1184, 256>>>(p0, p1, 64, n);      // first 64 rows: special-value families
    CK(cudaDeviceSynchronize());

    if (argc > 2 && !strcmp(argv[2], "ncu")) {     // profiling mode: a few launches of the candidate kernels only
        const __half* q0 = p0 + (size_t)64 * n;
        const __half* q1 = p1 + (size_t)64 * n;
        for (int i = 0; i < 3; ++i) {
            run_l2<256, false, true>(q0, q1, o1, 1984, n, 4, 0.4);
            run_l2<256, false, false>(q0, q1, o1, 1984, n, 4, 0.4);
        }
        CK(cudaDeviceSynchronize());
        return 0;
    }
    auto diff = [&](const char* name, int rows, int nn) {
        CK(cudaMemset(cnt, 0, 8));
        count_diff<<<1184, 256>>>((const uint16_t*)o0, (const uint16_t*)o1, (size_t)rows * nn, cnt);
        unsigned long long h; CK(cudaMemcpy(&h, cnt, 8, cudaMemcpyDeviceToHost));
        printf("{\"check\": \"%s\", \"rows\": %d, \"n\": %d, \"mismatching_elements\": %llu}\n", name, rows, nn, h);
    };
    // ---- bit-exactness: V0 (anchor) vs stage exact vs stage certified, several fracts, special + random rows
    const double fr[4] = {0.4, 0.0, 1.0, 0.8137};
    for (int k = 0; k < 4; ++k) {
        const int rows = 256;
        CK(cudaMemset(o0, 0, tot * 2)); CK(cudaMemset(o1, 0xff, tot * 2));
        run_v0(p0, p1, o0, rows, n, fr[k]);
        run_stage<512, true>(p0, p1, o1, rows, n, 4, fr[k]);
        diff("v0_vs_stage_exact", rows, n);
        run_stage<512, false>(p0, p1, o1, rows, n, 4, fr[k]);
        diff("v0_vs_stage_certified", rows, n);
        run_stage<256, false>(p0, p1, o1, rows, n, 8, fr[k]);
        diff("v0_vs_stage_certified_c8_t256", rows, n);
        run_l2<256, false, true>(p0, p1, o1, rows, n, 8, fr[k]);
        diff("v0_vs_l2_certified_c8_t256", rows, n);
        run_l2<512, false, false>(p0, p1, o1, rows, n, 4, fr[k]);
        diff("v0_vs_l2_certified_c4_t512", rows, n);
        run_l2<256, true, true>(p0, p1, o1, rows, n, 2, fr[k]);
        diff("v0_vs_l2_exact_c2_t256", rows, n);
    }
    {   // n = 16384 (512^2 latents), single-CTA "cluster"
        const int rows = 256, nn = 16384;
        run_v0(p0, p1, o0, rows, nn, 0.3);
        run_stage<512, false>(p0, p1, o1, rows, nn, 1, 0.3);
        diff("v0_vs_stage_certified_n16384_c1", rows, nn);
        run_stage<256, false>(p0, p1, o1, rows, nn, 2, 0.3);
        diff("v0_vs_stage_certified_n16384_c2", rows, nn);
        run_l2<256, false, true>(p0, p1, o1, rows, nn, 1, 0.3);
        diff("v0_vs_l2_certified_n16384_c1", rows, nn);
        run_l2<256, false, true>(p0, p1, o1, rows, nn, 4, 0.3);
        diff("v0_vs_l2_certified_n16384_c4", rows, nn);
    }
    {
        CK(cudaMemset(cnt, 0, 8));
        count_uncertified<<<1024, 256>>>(p0 + (size_t)64 * n, p1 + (size_t)64 * n, n, 0.4, cnt);
        unsigned long long h; CK(cudaMemcpy(&h, cnt, 8, cudaMemcpyDeviceToHost));
        printf("{\"stat\": \"uncertified_fraction_random_rows\", \"value\": %.6f}\n", (double)h / (1024.0 * n));
        CK(cudaMemset(cnt, 0, 8));
        count_uncertified<<<64, 256>>>(p0, p1, n, 0.4, cnt);
        CK(cudaMemcpy(&h, cnt, 8, cudaMemcpyDeviceToHost));
        printf("{\"stat\": \"uncertified_fraction_special_rows\", \"value\": %.6f}\n", (double)h / (64.0 * n));
    }
    // ---- timing (random rows only: skip the 64 special rows so the exact path rate is the typical one)
    const __half* q0 = p0 + (size_t)64 * n;
    const __half* q1 = p1 + (size_t)64 * n;
    auto report = [&](const char* name, int rows, int nn, float ms) {
        double gbs = (double)rows * nn * 6 / (ms * 1e-3) / 1e9;
        printf("{\"kernel\": \"%s\", \"rows\": %d, \"n\": %d, \"us\": %.2f, \"GBs\": %.1f, \"frac_of_measured_hbm\": %.3f}\n", name, rows, nn, ms * 1e3, gbs, gbs / peak);
        fflush(stdout);
    };
    for (int rows : {30, 210, 840, 1984}) {
        report("v0_regs_c8", rows, n, time_ms([&] { run_v0(q0, q1, o0, rows, n, 0.4); }));
        report("stage_cert_c4_t256", rows, n, time_ms([&] { run_stage<256, false>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c8_t256_hint", rows, n, time_ms([&] { run_l2<256, false, true>(q0, q1, o1, rows, n, 8, 0.4); }));
        report("l2_cert_c8_t256", rows, n, time_ms([&] { run_l2<256, false, false>(q0, q1, o1, rows, n, 8, 0.4); }));
        report("l2_cert_c4_t256_hint", rows, n, time_ms([&] { run_l2<256, false, true>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c4_t256_nohint", rows, n, time_ms([&] { run_l2<256, false, false>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c4_t256_hint_occ1536", rows, n, time_ms([&] { run_l2<256, false, true, 1536>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c4_t256_hint_occ1024", rows, n, time_ms([&] { run_l2<256, false, true, 1024>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c2_t256_hint_occ1024", rows, n, time_ms([&] { run_l2<256, false, true, 1024>(q0, q1, o1, rows, n, 2, 0.4); }));
        report("l2_cert_c2_t128_hint_occ1024", rows, n, time_ms([&] { run_l2<128, false, true, 1024>(q0, q1, o1, rows, n, 2, 0.4); }));
        report("l2_cert_c4_t128_hint_occ1280", rows, n, time_ms([&] { run_l2<128, false, true, 1280>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c4_t512_hint", rows, n, time_ms([&] { run_l2<512, false, true>(q0, q1, o1, rows, n, 4, 0.4); }));
        report("l2_cert_c2_t512_hint", rows, n, time_ms([&] { run_l2<512, false, true>(q0, q1, o1, rows, n, 2, 0.4); }));
        report("l2_cert_c2_t256_hint", rows, n, time_ms([&] { run_l2<256, false, true>(q0, q1, o1, rows, n, 2, 0.4); }));
        report("l2_cert_c8_t128_hint", rows, n, time_ms([&] { run_l2<128, false, true>(q0, q1, o1, rows, n, 8, 0.4); }));
        report("l2_exact_c8_t256_hint", rows, n, time_ms([&] { run_l2<256, true, true>(q0, q1, o1, rows, n, 8, 0.4); }));
    }
    for (int rows : {840, 7936}) {
        const int nn = 16384;
        report("v0_regs_c4", rows, nn, time_ms([&] { run_v0(q0, q1, o0, rows, nn, 0.4); }));
        report("stage_cert_c2_t256", rows, nn, time_ms([&] { run_stage<256, false>(q0, q1, o1, rows, nn, 2, 0.4); }));
        report("l2_cert_c1_t256_hint", rows, nn, time_ms([&] { run_l2<256, false, true>(q0, q1, o1, rows, nn, 1, 0.4); }));
        report("l2_cert_c2_t256_hint", rows, nn, time_ms([&] { run_l2<256, false, true>(q0, q1, o1, rows, nn, 2, 0.4); }));
        report("l2_cert_c4_t128_hint", rows, nn, time_ms([&] { run_l2<128, false, true>(q0, q1, o1, rows, nn, 4, 0.4); }));
        report("l2_cert_c1_t512_hint", rows, nn, time_ms([&] { run_l2<512, false, true>(q0, q1, o1, rows, nn, 1, 0.4); }));
    }
    return 0;
}
