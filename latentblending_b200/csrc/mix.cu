// mix.cu -- K1: latent mixing kernels (whole-row slerp, lerp).
//
// Replaces latentblending/utils.py:29-71 (interpolate_spherical), the
// per-branch parental-mix loop blending_engine.py:442-450 and the in-loop
// crossfeed diffusers_holder.py:322-324.  HBM-bound: 2 reads + 1 write per
// element (6 B/elem in fp16).
//
// Fast path (slerp_l2_kernel, mix_kernels.cuh): one thread-block CLUSTER per row.
// Pass 1 streams each CTA's slice of both inputs from HBM (L2 evict_last hint) into
// the three fp64 row reductions (|p0|^2, |p1|^2, <p0,p1>), combined across the cluster
// through distributed shared memory; the acos/sin weights are computed once per row and
// broadcast over DSMEM; pass 2 re-reads the slice from L2 (evict_first), evaluates the
// axpby with a certified fp32 fast path (exact fp64 fallback per element pair) and writes
// 128-bit streaming stores -- DRAM sees 2 reads + 1 write per element.
// Generic path (any n / alignment): partial-sum kernel + apply kernel through a
// small workspace; deterministic (fixed summation order, no atomics).
#include <stdlib.h>

#include "common.cuh"
#include "mix_kernels.cuh"

using namespace lbmix;

namespace {

constexpr int kThreads = 256;
constexpr int kParts = 8;  // partials per row in the generic path

// LB_SLERP_EXACT=1: evaluate pass 2 in fp64 for every element (the reference arithmetic verbatim) instead of the
// certified fp32 path -- same bits, used by the tests to A/B the certification.
bool lb_slerp_exact_pass2() {
    const char* e = getenv("LB_SLERP_EXACT");
    return e && e[0] == '1';
}

__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ void from_f(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void from_f(float* p, float v) { *p = v; }

__device__ __forceinline__ void block_reduce3(double& aa, double& bb, double& ab, double* sm /*[96]*/) {
    lbmix::block_reduce3<kThreads>(aa, bb, ab, sm);
}

// ---- generic path ---------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
slerp_partial_kernel(const T* __restrict__ p0, const T* __restrict__ p1, int64_t n, int64_t stride0,
                     int64_t stride1, double* __restrict__ partials) {
    pdl_launch_dependents();
    pdl_wait();
    const int64_t row = blockIdx.y;
    const T* a_row = p0 + row * stride0;
    const T* b_row = p1 + row * stride1;
    __shared__ double red[96];
    double aa = 0.0, bb = 0.0, ab = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)kParts * kThreads) {
        double da = to_f(a_row[i]), db = to_f(b_row[i]);
        aa = fma(da, da, aa);
        bb = fma(db, db, bb);
        ab = fma(da, db, ab);
    }
    block_reduce3(aa, bb, ab, red);
    if (threadIdx.x == 0) {
        double* dst = partials + (row * kParts + blockIdx.x) * 3;
        dst[0] = aa;
        dst[1] = bb;
        dst[2] = ab;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
slerp_apply_kernel(const T* __restrict__ p0, const T* __restrict__ p1, T* __restrict__ out, int64_t n,
                   int64_t stride0, int64_t stride1, int64_t stride_out, double fract,
                   const double* __restrict__ fract_rows, const double* __restrict__ partials) {
    pdl_launch_dependents();
    pdl_wait();
    const int64_t row = blockIdx.y;
    double aa = 0.0, bb = 0.0, ab = 0.0;
    for (int p = 0; p < kParts; ++p) {
        const double* src = partials + (row * kParts + p) * 3;
        aa += src[0];
        bb += src[1];
        ab += src[2];
    }
    double s0, s1;
    slerp_weights(aa, bb, ab, fract_rows ? fract_rows[row] : fract, s0, s1);
    const T* a_row = p0 + row * stride0;
    const T* b_row = p1 + row * stride1;
    T* o_row = out + row * stride_out;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
        from_f(o_row + i, slerp_elem(to_f(a_row[i]), to_f(b_row[i]), s0, s1));
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
lerp_kernel(const T* __restrict__ p0, const T* __restrict__ p1, T* __restrict__ out, int64_t n, float w0,
            float w1) {
    pdl_launch_dependents();
    pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        // torch: (1-f)*p0 -> store dtype; f*p1 -> store dtype; add -> store dtype
        T a, b;
        from_f(&a, w0 * to_f(p0[i]));
        from_f(&b, w1 * to_f(p1[i]));
        from_f(out + i, __fadd_rn(to_f(a), to_f(b)));
    }
}

// fast path launch: cluster of `csize` CTAs per row, `slice` elements of each input per CTA (two passes over
// global memory, the second served by L2 -- see slerp_l2_kernel).  Tuned with tools/ubench_mix.cu:
// 256 threads, 128 elements per thread and input, 4 CTAs resident per SM.
constexpr int kFastThreads = 256;
constexpr int kFastOcc = 1024;
constexpr int64_t kSliceElemsTarget = 32768;

template <typename T, bool EXACT2>
int launch_fast(const T* p0, const T* p1, T* out, int64_t rows, int64_t n, int64_t s0, int64_t s1, int64_t so,
                double fract, const double* fract_rows, int csize, int slice, cudaStream_t st) {
    auto kern = slerp_l2_kernel<T, kFastThreads, EXACT2, true, kFastOcc>;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)csize, (unsigned)rows, 1);
    cfg.blockDim = dim3(kFastThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)csize;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = lb_pdl_enabled() ? 2 : 1;
    LB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, p0, p1, out, n, slice, s0, s1, so, fract, fract_rows));
    return 0;
}

template <typename T>
int slerp_dispatch(const void* p0v, const void* p1v, void* outv, int64_t rows, int64_t n, int64_t s0,
                   int64_t s1, int64_t so, double fract, const double* fract_rows, void* ws, cudaStream_t st) {
    const T* p0 = static_cast<const T*>(p0v);
    const T* p1 = static_cast<const T*>(p1v);
    T* out = static_cast<T*>(outv);
    constexpr int VE = Vec<T>::N;
    const bool vec_ok = (n % VE == 0) && (s0 % VE == 0) && (s1 % VE == 0) && (so % VE == 0) &&
                        lb_aligned16(p0) && lb_aligned16(p1) && lb_aligned16(out);
    if (vec_ok && rows <= 65535 && n <= (int64_t)1 << 30) {
        // smallest power-of-two cluster (<= 8, the portable limit) whose slices are <= the target
        int csize = 1;
        while (csize < 8 && lb_ceil_div(n, csize) > kSliceElemsTarget) csize *= 2;
        const int64_t slice = lb_ceil_div(lb_ceil_div(n, csize), VE) * VE;
        if (sizeof(T) == 2 && !lb_slerp_exact_pass2())
            return launch_fast<T, false>(p0, p1, out, rows, n, s0, s1, so, fract, fract_rows, csize, (int)slice, st);
        return launch_fast<T, true>(p0, p1, out, rows, n, s0, s1, so, fract, fract_rows, csize, (int)slice, st);
    }
    LB_REQUIRE(ws != nullptr, "lb_slerp_rows: generic path needs the workspace");
    LB_REQUIRE(rows <= 65535, "lb_slerp_rows: rows > 65535 unsupported");
    double* partials = static_cast<double*>(ws);
    lb_launch_pdl(slerp_partial_kernel<T>, dim3(kParts, (unsigned)rows), kThreads, 0, st, p0, p1, n, s0, s1, partials);
    LB_LAUNCH_CHECK();
    unsigned gx = (unsigned)lb_ceil_div(n, (int64_t)kThreads * 8);
    if (gx < 1) gx = 1;
    if (gx > 1024) gx = 1024;
    lb_launch_pdl(slerp_apply_kernel<T>, dim3(gx, (unsigned)rows), kThreads, 0, st, p0, p1, out, n, s0, s1, so, fract,
                                                                         fract_rows, partials);
    LB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" size_t lb_slerp_workspace_bytes(int64_t rows, int64_t /*n*/) {
    return (size_t)rows * kParts * 3 * sizeof(double);
}

extern "C" int lb_slerp_rows(lb_ctx* ctx, const void* p0, const void* p1, void* out, int64_t rows, int64_t n,
                             int64_t stride0, int64_t stride1, int64_t stride_out, int dtype, double fract,
                             const double* fract_rows_dev, void* workspace_dev, void* stream) {
    LB_REQUIRE(ctx != nullptr, "lb_slerp_rows: null context");
    LB_REQUIRE(rows >= 0 && n >= 0, "lb_slerp_rows: negative size");
    if (rows == 0 || n == 0) return 0;
    LB_REQUIRE(p0 && p1 && out, "lb_slerp_rows: null buffer");
    LB_REQUIRE(dtype == 0 || dtype == 1, "lb_slerp_rows: dtype must be 0 (fp16) or 1 (fp32)");
    cudaStream_t st = lb_stream(stream);
    if (dtype == 0)
        return slerp_dispatch<__half>(p0, p1, out, rows, n, stride0, stride1, stride_out, fract, fract_rows_dev,
                                      workspace_dev, st);
    return slerp_dispatch<float>(p0, p1, out, rows, n, stride0, stride1, stride_out, fract, fract_rows_dev,
                                 workspace_dev, st);
}

extern "C" int lb_lerp(lb_ctx* ctx, const void* p0, const void* p1, void* out, int64_t n, int dtype,
                       double fract, void* stream) {
    LB_REQUIRE(ctx != nullptr, "lb_lerp: null context");
    if (n == 0) return 0;
    LB_REQUIRE(p0 && p1 && out, "lb_lerp: null buffer");
    LB_REQUIRE(dtype == 0 || dtype == 1, "lb_lerp: dtype must be 0 (fp16) or 1 (fp32)");
    const float w0 = (float)(1.0 - fract), w1 = (float)fract;
    unsigned grid = (unsigned)lb_ceil_div(n, kThreads * 4);
    if (grid > (unsigned)ctx->sm_count * 8) grid = (unsigned)ctx->sm_count * 8;
    if (grid < 1) grid = 1;
    cudaStream_t st = lb_stream(stream);
    if (dtype == 0)
        lb_launch_pdl(lerp_kernel<__half>, grid, kThreads, 0, st, (const __half*)p0, (const __half*)p1, (__half*)out, n, w0, w1);
    else
        lb_launch_pdl(lerp_kernel<float>, grid, kThreads, 0, st, (const float*)p0, (const float*)p1, (float*)out, n, w0, w1);
    LB_LAUNCH_CHECK();
    return 0;
}
