// mix_kernels.cuh -- device code of K1 (whole-row slerp).  Included by mix.cu (the C ABI) and by
// tools/ubench_mix.cu (stand-alone micro-benchmark of the variants).
//
// Arithmetic contract = latentblending/utils.py:29-71 (interpolate_spherical):
//   p0,p1 -> fp64; aa = sum p0^2, bb = sum p1^2, ab = sum p0*p1 (fp64);
//   dot = clamp(ab / (sqrt(aa) sqrt(bb)), -1+1e-7, 1-1e-7); theta0 = acos(dot);
//   s0 = sin(theta0 - theta0*f)/sin(theta0); s1 = sin(theta0*f)/sin(theta0);
//   out = (storage dtype)(float)(p0*s0 + p1*s1)         [fp64 mul, mul, add, no FMA contraction]
//
// Two single-DRAM-pass designs live here (both bit-identical to the all-fp64 evaluation; tools/ubench_mix.cu
// compares them):
//   slerp_l2_kernel    (the product path): pass 1 streams the row slice from HBM, pass 2 re-reads it from L2.
//                      No on-chip staging -> ~48 registers, 4-6 CTAs per SM hide the serial section of each CTA
//                      (row reduction -> cluster exchange -> acos/sin weights).
//   slerp_stage_kernel (kept as the measured alternative): cp.async.bulk stages the slice in shared memory once.
//                      Exact 6 B/elem DRAM traffic, but only 3 CTAs fit per SM.
// Pass 2 (the axpby): the reference evaluates it in fp64 and rounds fp64 -> fp32 -> fp16; doing that per element
// costs 3 fp64 conversions + 3 fp64 ops and makes the kernel XU/fp64-pipe-bound (round-1a kernel: 2.1 TB/s).
// Instead each element is evaluated in packed fp32 with the weights split hi+lo and the fp16 rounding is
// CERTIFIED (derivation at slerp_vec8_h): if the fp32 value is farther from every fp16 rounding boundary than
// the proven error bound, rounding it gives bit-for-bit the reference result; otherwise (~0.1 % of elements,
// subnormal / overflowing results, NaN/Inf) that element pair takes the exact fp64 path.
#pragma once
#include <cooperative_groups.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace lbmix {

namespace cg = cooperative_groups;

constexpr double kClampEps = 1e-7;  // utils.py:55

// ---- element packing -------------------------------------------------------------------
template <typename T> struct Vec;
template <> struct Vec<__half> {
    static constexpr int N = 8;
    __device__ static void unpack(const uint4& v, float (&f)[8]) {
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float2 t = __half22float2(h[i]);
            f[2 * i] = t.x;
            f[2 * i + 1] = t.y;
        }
    }
    __device__ static uint4 pack(const float (&f)[8]) {
        uint4 v;
        __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        return v;
    }
};
template <> struct Vec<float> {
    static constexpr int N = 4;
    __device__ static void unpack(const uint4& v, float (&f)[4]) {
        f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
        f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
    }
    __device__ static uint4 pack(const float (&f)[4]) {
        return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                          __float_as_uint(f[3]));
    }
};

// utils.py:54-63 in fp64: the two slerp weights from the three row sums.
__device__ __forceinline__ void slerp_weights(double aa, double bb, double ab, double fract, double& s0,
                                              double& s1) {
    double norm = sqrt(aa) * sqrt(bb);
    double dot = ab / norm;
    dot = fmin(fmax(dot, -1.0 + kClampEps), 1.0 - kClampEps);
    double theta0 = acos(dot);
    double sin0 = sin(theta0);
    double theta_t = theta0 * fract;
    s0 = sin(theta0 - theta_t) / sin0;
    s1 = sin(theta_t) / sin0;
}

// fp64 axpby without FMA contraction (torch: mul, mul, add), then the reference's fp64 -> fp32 cast
// (the storage-dtype cast follows at the call site).
__device__ __forceinline__ float slerp_elem(float a, float b, double s0, double s1) {
    double r = __dadd_rn(__dmul_rn((double)a, s0), __dmul_rn((double)b, s1));
    return __double2float_rn(r);
}

// fp64 weight split into fp32 hi + lo (|s - hi - lo| <= 2^-48 |s|) plus the error-bound coefficients
struct SplitW {
    float s0h, s0l, s1h, s1l, e1;
    __device__ SplitW() {}
    __device__ SplitW(double s0, double s1) {
        s0h = __double2float_rn(s0);
        s0l = __double2float_rn(s0 - (double)s0h);
        s1h = __double2float_rn(s1);
        s1l = __double2float_rn(s1 - (double)s1h);
        e1 = fabsf(s1h) * kErrB;
    }
    static constexpr float kErrR = 1.0625f * 1.1920928955078125e-07f;   // 1.0625 * 2^-23  (coefficient of |r|)
    static constexpr float kErrB = 1.0625f * 5.9604644775390625e-08f;   // 1.0625 * 2^-24  (coefficient of |b s1h|)
};

// ---- certified fp32 evaluation of (half)(float)(fp64(a)*s0 + fp64(b)*s1) for fp16-valued a, b -------------
//   r  = fl(a s0h + t3), t3 = fl(b s1h + t2), t2 = fl(a s0l + t1), t1 = fl(b s1l)       (fp32, 4 operations)
// Error vs the exact real x = a s0 + b s1, with M = |a s0| + |b s1|:
//   |t1 - b s1l| <= 2^-48 |b s1|;  |t2 - (a s0l + t1)| <= 2^-24 |t2| <= 2^-48 M (1+e);
//   |t3 - (b s1h + t2)| <= 2^-24 |t3| <= 2^-24 |b s1h| + 2^-48 M;   |r - (a s0h + t3)| <= 2^-24 |r|;
//   the split itself loses <= 2^-48 M   =>   |r - x| <= B := 2^-24 (|r| + |b s1h|) + 2^-45 M,
//   and M <= |r| + 2 |b s1h| (1+e) makes the last term < 2^-20 of the first.  The reference's fp64 value R
//   (two products and a sum, each rounded) has |R - x| <= 2^-51 M.
// Rounding: the reference returns RN16(RN32(R)).  Let mid be the fp16 rounding midpoint nearest to r, at distance
//   m; u = half the fp16 spacing in r's binade; d = |r - RN16(r)| = u - m.  If m > B + ulp32(r)/2 then R is on
//   r's side of mid AND farther than half an fp32 ulp from it, so RN32(R) is on that side too (never ON mid: no
//   tie), hence RN16(RN32(R)) = RN16(r).  With ulp32(r)/2 <= 2^-24 |r| the test uses
//       E = 1.0625 * 2^-24 * (2 |r| + |b s1h|)   >=  B + ulp32(r)/2   (6 % slack covers E's own two roundings)
//       certified  <=>  E + max(d, E) < u         (d >= E: m = u - d > E;   d < E: 2E < u)
//   2E < u also covers R and r straddling a power of two (finer grid below it): |R - 2^k| <= E < u/2 rounds to 2^k.
//   No range test is needed: for |r| < 2^-14 (fp16 subnormals, coarser grid) u only gets stricter and turns negative
//   below 2^-116; r >= 65520 rounds to inf so d = inf; NaN fails every comparison.  Uncertified elements (~0.1 %)
//   are recomputed with the reference's fp64 arithmetic, so the output is bit-identical to the all-fp64 evaluation.
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
// scalar form (used by the statistics kernel of tools/ubench_mix.cu; same arithmetic as the packed form)
__device__ __forceinline__ float slerp_fast(float a, float b, const SplitW& w, float& E) {
    float t = b * w.s1l;
    t = fmaf(a, w.s0l, t);
    t = fmaf(b, w.s1h, t);
    const float r = fmaf(a, w.s0h, t);
    E = fmaf(fabsf(b), w.e1, fabsf(r) * SplitW::kErrR);
    return r;
}
__device__ __forceinline__ bool slerp_certified_d(float r, float diff, float E) {   // diff = r - RN16(r)
    const float u = __uint_as_float((__float_as_uint(r) & 0x7f800000u) - (11u << 23));   // 2^(e-11)
    return E + fmaxf(fabsf(diff), E) < u;
}
__device__ __forceinline__ bool slerp_certified(float r, float back, float E) {
    const float d = fabsf(r - back);
    const float u = __uint_as_float((__float_as_uint(r) & 0x7f800000u) - (11u << 23));   // 2^(e-11)
    return E + fmaxf(d, E) < u;
}
// exact path, kept out of line so the certified loop stays branch-over (not predicated fp64 code)
__device__ __noinline__ uint32_t slerp_exact_bits(float a, float b, double s0, double s1) {
    return (uint32_t)__half_as_ushort(__float2half_rn(slerp_elem(a, b, s0, s1)));
}
// 8 elements (one 128-bit vector of each input) -> 8 fp16 results; packed fp32 math, ONE branch per vector
__device__ __forceinline__ uint4 slerp_vec8_h(const uint4& ua, const uint4& ub, const SplitW& w, double s0,
                                              double s1) {
    const __half2* ha = reinterpret_cast<const __half2*>(&ua);
    const __half2* hb = reinterpret_cast<const __half2*>(&ub);
    const float2 s0h = make_float2(w.s0h, w.s0h), s0l = make_float2(w.s0l, w.s0l);
    const float2 s1h = make_float2(w.s1h, w.s1h), s1l = make_float2(w.s1l, w.s1l);
    const float2 kr2 = make_float2(SplitW::kErrR, SplitW::kErrR), neg1 = make_float2(-1.f, -1.f);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
    bool okp[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 a = __half22float2(ha[i]);
        const float2 b = __half22float2(hb[i]);
        float2 t = mul2(b, s1l);
        t = fma2(a, s0l, t);
        t = fma2(b, s1h, t);
        const float2 r = fma2(a, s0h, t);
        const __half2 h = __floats2half2_rn(r.x, r.y);
        const float2 back = __half22float2(h);
        ow[i] = *reinterpret_cast<const uint32_t*>(&h);
        const float2 rk = mul2(r, kr2);                       // |rk| = |r| * kErrR (exact scaling by 1.0625 * 2^-23 up to 1 rounding)
        const float2 dd = fma2(back, neg1, r);                // r - back, exact
        const float E0 = fmaf(fabsf(b.x), w.e1, fabsf(rk.x));
        const float E1 = fmaf(fabsf(b.y), w.e1, fabsf(rk.y));
        okp[i] = slerp_certified_d(r.x, dd.x, E0) & slerp_certified_d(r.y, dd.y, E1);   // no short-circuit
    }
    if (!((okp[0] & okp[1]) & (okp[2] & okp[3]))) {
        // about a fifth of the warp-vectors hold an uncertified element: that PAIR is recomputed with the reference's
        // fp64 arithmetic (both halves -- cheaper than re-testing which one failed)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (!okp[i]) {
                const float2 a = __half22float2(ha[i]);
                const float2 b = __half22float2(hb[i]);
                ow[i] = slerp_exact_bits(a.x, b.x, s0, s1) | (slerp_exact_bits(a.y, b.y, s0, s1) << 16);
            }
        }
    }
    return o;
}

// fp16 -> fp64 in ONE conversion (cvt.f64.f16), both halves of a packed pair
__device__ __forceinline__ void h2_to_d2(uint32_t packed, double& lo, double& hi) {
    asm("{\n\t.reg .b16 l, h;\n\t"
        "mov.b32 {l, h}, %2;\n\t"
        "cvt.f64.f16 %0, l;\n\t"
        "cvt.f64.f16 %1, h;\n\t}"
        : "=d"(lo), "=d"(hi)
        : "r"(packed));
}
template <typename T> struct ToD;
template <> struct ToD<__half> {     // uint4 = 8 halves
    __device__ static void cvt(const uint4& v, double (&d)[8]) {
        h2_to_d2(v.x, d[0], d[1]);
        h2_to_d2(v.y, d[2], d[3]);
        h2_to_d2(v.z, d[4], d[5]);
        h2_to_d2(v.w, d[6], d[7]);
    }
};
template <> struct ToD<float> {      // uint4 = 4 floats
    __device__ static void cvt(const uint4& v, double (&d)[4]) {
        d[0] = (double)__uint_as_float(v.x);
        d[1] = (double)__uint_as_float(v.y);
        d[2] = (double)__uint_as_float(v.z);
        d[3] = (double)__uint_as_float(v.w);
    }
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum of three doubles; result valid in every thread.  sm: [3 * 32] doubles.
template <int THREADS>
__device__ __forceinline__ void block_reduce3(double& aa, double& bb, double& ab, double* sm) {
    constexpr int W = THREADS / 32;
    aa = warp_sum_d(aa);
    bb = warp_sum_d(bb);
    ab = warp_sum_d(ab);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) {
        sm[w] = aa;
        sm[32 + w] = bb;
        sm[64 + w] = ab;
    }
    __syncthreads();
    aa = bb = ab = 0.0;
#pragma unroll
    for (int i = 0; i < W; ++i) {
        aa += sm[i];
        bb += sm[32 + i];
        ab += sm[64 + i];
    }
}

// ---- async bulk copy (TMA 1-D) + mbarrier ----------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}
__device__ __forceinline__ void bar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void bar_expect(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n\t.reg .pred P;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, P;\n\t}"
            : "=r"(ok)
            : "r"(smem_addr(bar)), "r"(parity)
            : "memory");
    }
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void stg_stream(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- fast path --------------------------------------------------------------------------------
// grid (csize, rows), cluster (csize,1,1).  `slice` = elements per CTA (multiple of Vec<T>::N; the last CTA of a
// row may own fewer).  Dynamic smem: 2 * slice * sizeof(T) (16 B aligned).  EXACT2 = evaluate pass 2 in fp64 for
// every element (reference arithmetic verbatim; used for fp32 storage and as the A/B check of the certified path).
template <typename T, int THREADS, bool EXACT2>
__global__ void __launch_bounds__(THREADS)
slerp_stage_kernel(const T* __restrict__ p0, const T* __restrict__ p1, T* __restrict__ out, int64_t n, int slice,
                   int64_t stride0, int64_t stride1, int64_t stride_out, double fract,
                   const double* __restrict__ fract_rows) {
    griddep_launch_dependents();
    constexpr int VE = Vec<T>::N;
    extern __shared__ __align__(128) uint8_t stage_raw[];
    __shared__ double red[96];
    __shared__ double cta_sum[3];
    __shared__ __align__(8) uint64_t bar;

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned crank = cluster.block_rank();
    const unsigned csize = cluster.num_blocks();
    const int64_t row = blockIdx.y;
    const int64_t e0 = (int64_t)crank * slice;                       // first element of this CTA's slice
    const int mine = (int)max((int64_t)0, min((int64_t)slice, n - e0));   // elements this CTA owns
    const uint32_t bytes = (uint32_t)mine * (uint32_t)sizeof(T);
    T* sa = reinterpret_cast<T*>(stage_raw);
    T* sb = reinterpret_cast<T*>(stage_raw + (size_t)slice * sizeof(T));

    if (threadIdx.x == 0) bar_init(&bar, 1);
    __syncthreads();
    griddep_wait();                                                   // inputs may be the previous kernel's output
    if (threadIdx.x == 0) {
        bar_expect(&bar, 2 * bytes);
        if (bytes) {
            bulk_g2s(sa, p0 + row * stride0 + e0, bytes, &bar);
            bulk_g2s(sb, p1 + row * stride1 + e0, bytes, &bar);
        }
    }
    bar_wait(&bar, 0);

    // ---- pass 1: fp64 row sums (two interleaved accumulator sets shorten the DFMA chains)
    const int nvec = mine / VE;
    double aa0 = 0.0, bb0 = 0.0, ab0 = 0.0, aa1 = 0.0, bb1 = 0.0, ab1 = 0.0;
    for (int v = threadIdx.x; v < nvec; v += THREADS) {
        double da[VE], db[VE];
        ToD<T>::cvt(reinterpret_cast<const uint4*>(sa)[v], da);
        ToD<T>::cvt(reinterpret_cast<const uint4*>(sb)[v], db);
#pragma unroll
        for (int e = 0; e < VE; e += 2) {
            const double da0 = da[e], db0 = db[e], da1 = da[e + 1], db1 = db[e + 1];
            aa0 = fma(da0, da0, aa0);
            bb0 = fma(db0, db0, bb0);
            ab0 = fma(da0, db0, ab0);
            aa1 = fma(da1, da1, aa1);
            bb1 = fma(db1, db1, bb1);
            ab1 = fma(da1, db1, ab1);
        }
    }
    double aa = aa0 + aa1, bb = bb0 + bb1, ab = ab0 + ab1;
    block_reduce3<THREADS>(aa, bb, ab, red);
    if (threadIdx.x == 0) {
        cta_sum[0] = aa;
        cta_sum[1] = bb;
        cta_sum[2] = ab;
    }
    cluster_arrive();
    cluster_wait();
    double taa = 0.0, tbb = 0.0, tab = 0.0;
    for (unsigned r = 0; r < csize; ++r) {
        const double* remote = cluster.map_shared_rank(cta_sum, r);
        taa += remote[0];
        tbb += remote[1];
        tab += remote[2];
    }
    cluster_arrive();          // peers may exit once everybody has read their cta_sum (waited for at the end)
    const double f = fract_rows ? fract_rows[row] : fract;
    double s0, s1;
    slerp_weights(taa, tbb, tab, f, s0, s1);
    const SplitW w(s0, s1);

    // ---- pass 2: axpby from smem, 128-bit coalesced stores
    T* o_row = out + row * stride_out + e0;
    for (int v = threadIdx.x; v < nvec; v += THREADS) {
        const uint4 ua = reinterpret_cast<const uint4*>(sa)[v];
        const uint4 ub = reinterpret_cast<const uint4*>(sb)[v];
        uint4 o;
        if constexpr (!EXACT2 && sizeof(T) == 2) {
            o = slerp_vec8_h(ua, ub, w, s0, s1);
        } else {
            float fa[VE], fb[VE], fo[VE];
            Vec<T>::unpack(ua, fa);
            Vec<T>::unpack(ub, fb);
#pragma unroll
            for (int e = 0; e < VE; ++e) fo[e] = slerp_elem(fa[e], fb[e], s0, s1);
            o = Vec<T>::pack(fo);
        }
        stg_stream(o_row + (int64_t)v * VE, o);
    }
    cluster_wait();
}

// ---- fast path B: two passes over global memory, the second served by L2 ------------------------
// No on-chip staging at all: pass 1 streams the CTA's slice of both inputs from HBM (fp64 sums), pass 2 reads the
// same slice again a few microseconds later -- by then it is resident in L2 (a whole launch keeps
// < 132 SMs x 8 CTAs x 64 KiB = 68 MB in flight, against the H100's 50 MB L2 the oldest slices may be evicted), so DRAM still sees 2 reads + 1 write per element.  With ~40
// registers per thread and no shared-memory footprint, 8 CTAs are resident per SM and the long serial section
// of each CTA (row reduction -> cluster exchange -> acos/sin weights -> second pass) is hidden by the others.
// The weights are computed ONCE per row (rank 0, warp 0) and broadcast through distributed shared memory.
struct RowWeights {
    double s0, s1;
    float s0h, s0l, s1h, s1l, e1, pad;
};

__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// first read of a line: it will be read once more by this CTA a few microseconds later -> keep it in L2
template <bool HINT>
__device__ __forceinline__ uint4 ldg_pass1(const void* p, uint64_t pol) {
    uint4 r;
    if constexpr (HINT)
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    else
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
template <bool HINT>
__device__ __forceinline__ void stg_hint(void* p, const uint4& v, uint64_t pol) {
    if constexpr (HINT)
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x),
                     "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol)
                     : "memory");
    else
        stg_stream(p, v);
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// second (last) read of a line: tell L2 it is the first candidate for replacement
template <bool HINT>
__device__ __forceinline__ uint4 ldg_pass2(const void* p, uint64_t pol) {
    uint4 r;
    if constexpr (HINT)
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    else
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

template <typename T, int THREADS, bool EXACT2, bool HINT, int OCC = 1280>
__global__ void __launch_bounds__(THREADS, OCC / THREADS)
slerp_l2_kernel(const T* __restrict__ p0, const T* __restrict__ p1, T* __restrict__ out, int64_t n, int slice,
                int64_t stride0, int64_t stride1, int64_t stride_out, double fract,
                const double* __restrict__ fract_rows) {
    griddep_launch_dependents();
    constexpr int VE = Vec<T>::N;
    __shared__ double red[96];
    __shared__ double cta_sum[3];
    __shared__ RowWeights wbuf;

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned crank = cluster.block_rank();
    const unsigned csize = cluster.num_blocks();
    const int64_t row = blockIdx.y;
    const int64_t e0 = (int64_t)crank * slice;
    const int mine = (int)max((int64_t)0, min((int64_t)slice, n - e0));
    const int nvec = mine / VE;
    const uint4* a4 = reinterpret_cast<const uint4*>(p0 + row * stride0 + e0);
    const uint4* b4 = reinterpret_cast<const uint4*>(p1 + row * stride1 + e0);
    uint4* o4 = reinterpret_cast<uint4*>(out + row * stride_out + e0);
    griddep_wait();

    // ---- pass 1 (HBM): fp64 row sums
    const uint64_t pol_keep = l2_policy_evict_last();
    double aa0 = 0.0, bb0 = 0.0, ab0 = 0.0, aa1 = 0.0, bb1 = 0.0, ab1 = 0.0;
#pragma unroll 4
    for (int v = threadIdx.x; v < nvec; v += THREADS) {
        double da[VE], db[VE];
        ToD<T>::cvt(ldg_pass1<HINT>(a4 + v, pol_keep), da);
        ToD<T>::cvt(ldg_pass1<HINT>(b4 + v, pol_keep), db);
#pragma unroll
        for (int e = 0; e < VE; e += 2) {
            aa0 = fma(da[e], da[e], aa0);
            bb0 = fma(db[e], db[e], bb0);
            ab0 = fma(da[e], db[e], ab0);
            aa1 = fma(da[e + 1], da[e + 1], aa1);
            bb1 = fma(db[e + 1], db[e + 1], bb1);
            ab1 = fma(da[e + 1], db[e + 1], ab1);
        }
    }
    double aa = aa0 + aa1, bb = bb0 + bb1, ab = ab0 + ab1;
    block_reduce3<THREADS>(aa, bb, ab, red);
    if (threadIdx.x == 0) {
        cta_sum[0] = aa;
        cta_sum[1] = bb;
        cta_sum[2] = ab;
    }
    cluster_arrive();
    cluster_wait();
    if (crank == 0 && threadIdx.x < 32) {
        // fixed-order combine, then the scalar fp64 section once per row
        double taa = 0.0, tbb = 0.0, tab = 0.0;
        for (unsigned r = 0; r < csize; ++r) {
            const double* remote = cluster.map_shared_rank(cta_sum, r);
            taa += remote[0];
            tbb += remote[1];
            tab += remote[2];
        }
        const double f = fract_rows ? fract_rows[row] : fract;
        RowWeights rw;
        slerp_weights(taa, tbb, tab, f, rw.s0, rw.s1);
        const SplitW w(rw.s0, rw.s1);
        rw.s0h = w.s0h; rw.s0l = w.s0l; rw.s1h = w.s1h; rw.s1l = w.s1l; rw.e1 = w.e1; rw.pad = 0.f;
        if (threadIdx.x < csize) *cluster.map_shared_rank(&wbuf, threadIdx.x) = rw;
    }
    cluster_arrive();
    cluster_wait();
    const double s0 = wbuf.s0, s1 = wbuf.s1;
    SplitW w;
    w.s0h = wbuf.s0h; w.s0l = wbuf.s0l; w.s1h = wbuf.s1h; w.s1l = wbuf.s1l; w.e1 = wbuf.e1;

    // ---- pass 2 (L2): axpby, 128-bit coalesced streaming stores
    const uint64_t pol = l2_policy_evict_first();
#pragma unroll 2
    for (int v = threadIdx.x; v < nvec; v += THREADS) {
        const uint4 ua = ldg_pass2<HINT>(a4 + v, pol);
        const uint4 ub = ldg_pass2<HINT>(b4 + v, pol);
        uint4 o;
        if constexpr (!EXACT2 && sizeof(T) == 2) {
            o = slerp_vec8_h(ua, ub, w, s0, s1);
        } else {
            float fa[VE], fb[VE], fo[VE];
            Vec<T>::unpack(ua, fa);
            Vec<T>::unpack(ub, fb);
#pragma unroll
            for (int e = 0; e < VE; ++e) fo[e] = slerp_elem(fa[e], fb[e], s0, s1);
            o = Vec<T>::pack(fo);
        }
        stg_hint<HINT>(o4 + v, o, pol);
    }
}

}  // namespace lbmix
