// norm.cu -- K5 GroupNorm(+SiLU) and K6 LayerNorm on NHWC fp16 activations.
//
// Replace torch.nn.GroupNorm (+ F.silu) in the UNet resnets / transformer entry /
// conv_norm_out and torch.nn.LayerNorm in the 70 transformer blocks (call site
// latentblending/diffusers_holder.py:336-344).  HBM/L2-bound: GroupNorm reads x
// twice (stats pass, apply pass -- the second read is an L2 hit for every SDXL
// activation) and writes once; LayerNorm is single-read (row kept in registers).
// Deterministic and batch-invariant: fixed-order reductions, no floating-point atomics (one integer
// "last block" counter per batch element finalises the statistics).  GroupNorm statistics are fp32 sums of x - K_g
// (K_g: a pilot value of the group, so E[x^2] - mean^2 does not cancel when the mean is large next to sigma), fp64
// final combine; output rounded to fp16 after the affine and again after SiLU, like the
// reference's two separate torch ops.  GroupNorm also exists in bf16 (the bf16 VAE decoder): same statistics and
// summation order, bf16 loads and roundings.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxC = 2560;

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

// ---- GroupNorm ----------------------------------------------------------------------------------
// Thread layout shared by both passes: a thread owns ONE 16-byte channel vector (8 channels) and walks rows;
// VP = C/8 vectors per row, RL = 256 / VP row lanes per block (C = 320: 6 lanes x 40 vectors).  All global
// accesses are 128-bit and coalesced along C, 4 rows in flight per thread, no integer divisions in the loops.
// The row-chunk grid depends on HW only (not on the batch), so results are bit-identical for any batch size.

// pass 1: per (batch, row-chunk) partial sums per group; the last chunk of a batch element to finish turns the
// partials into (mean, rstd) per group -- fixed summation order, fp64 combine, no floating-point atomics.
// The sums are shifted: S1 = sum (x - K_g), S2 = sum (x - K_g)^2 with K_g = x[b, row 0, first channel of group g], so
// mean = K_g + S1/n and var = S2/n - (S1/n)^2 lose no precision to a mean that is large next to sigma (unshifted fp32
// sums of x and x^2 put an error of order 2^-24 mean^2 into the variance).  The pilot is per image, so results stay
// batch-invariant.
template <typename T>
__global__ void __launch_bounds__(kThreads)
gn_partial_kernel(const T* __restrict__ x, long long ld, int C, int HW, int groups, int rows_per_chunk,
                  float eps, float2* __restrict__ partial /*[B][chunks][groups]*/,
                  float2* __restrict__ stats /*[B][groups] (mean, rstd)*/, int* __restrict__ counter /*[B]*/) {
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.y, chunk = blockIdx.x, chunks = gridDim.x;
    const int row0 = chunk * rows_per_chunk;
    const int row1 = min(HW, row0 + rows_per_chunk);
    const int VP = C >> 3;
    const int cpg = C / groups;
    __shared__ float s_sum[kMaxC], s_sq[kMaxC];
    __shared__ int s_last;
    for (int c = threadIdx.x; c < C; c += kThreads) s_sum[c] = s_sq[c] = 0.f;
    __syncthreads();
    const T* base = x + ((long long)b * HW) * ld;
    const int RL = VP <= kThreads ? kThreads / VP : 1;
    for (int cv0 = 0; cv0 < VP; cv0 += kThreads) {          // one trip unless C > 2048
        const int cv = cv0 + (VP <= kThreads ? (int)threadIdx.x % VP : (int)threadIdx.x);
        const int rl = VP <= kThreads ? (int)threadIdx.x / VP : 0;
        const bool active = cv < VP && rl < RL;
        float s[8], q[8], k[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = q[j] = k[j] = 0.f;
        if (active) {
            const T* col = base + 8 * cv;
#pragma unroll
            for (int j = 0; j < 8; ++j) k[j] = LbType<T>::to_f(base[(8 * cv + j) / cpg * cpg]);    // K_g of channel
#pragma unroll 4
            for (int r = row0 + rl; r < row1; r += RL) {
                const uint4 v = *reinterpret_cast<const uint4*>(col + (long long)r * ld);
                const auto* h = reinterpret_cast<const typename LbType<T>::T2*>(&v);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = LbType<T>::to_f2(h[j]);
                    const float d0 = f.x - k[2 * j], d1 = f.y - k[2 * j + 1];
                    s[2 * j] += d0;
                    s[2 * j + 1] += d1;
                    q[2 * j] = fmaf(d0, d0, q[2 * j]);
                    q[2 * j + 1] = fmaf(d1, d1, q[2 * j + 1]);
                }
            }
        }
        // combine the row lanes in lane order (deterministic); every thread reaches every barrier
        for (int l = 0; l < RL; ++l) {
            if (active && rl == l) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    s_sum[8 * cv + j] += s[j];
                    s_sq[8 * cv + j] += q[j];
                }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x < groups) {
        const int g = threadIdx.x;
        float s = 0.f, q = 0.f;
        for (int i = 0; i < cpg; ++i) {
            s += s_sum[g * cpg + i];
            q += s_sq[g * cpg + i];
        }
        partial[((long long)b * chunks + chunk) * groups + g] = make_float2(s, q);
    }
    // last chunk of this batch element finalises the statistics
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&counter[b], 1) == chunks - 1);
    __syncthreads();
    if (s_last) {
        __threadfence();
        // All 256 threads of the last block combine the chunk partials: thread (slice, g) sums chunks slice, slice + S,
        // ... of group g in fp64 with 8 loads in flight, then the S slices are added in slice order -- a fixed
        // summation order (deterministic, batch-invariant).  One thread per group walking all ~300 chunks was a serial
        // chain of L2 round trips: ~20 us, most of this kernel's time on the large activations.
        __shared__ double f_sum[kThreads], f_sq[kThreads];
        const int S = kThreads / groups;                 // slices (groups <= 64 -> S >= 4)
        const int g = threadIdx.x % groups, slice = threadIdx.x / groups;
        double s = 0.0, q = 0.0;
        if (slice < S) {
            const float2* pp = partial + (long long)b * chunks * groups + g;
            for (int c0 = slice; c0 < chunks; c0 += 8 * S) {
                float2 v[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int c = c0 + i * S;
                    v[i] = c < chunks ? __ldcg(pp + (long long)c * groups) : make_float2(0.f, 0.f);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    s += v[i].x;
                    q += v[i].y;
                }
            }
        }
        f_sum[threadIdx.x] = s;
        f_sq[threadIdx.x] = q;
        __syncthreads();
        if (threadIdx.x < groups) {
            double ts = 0.0, tq = 0.0;
            for (int sl = 0; sl < S; ++sl) {
                ts += f_sum[sl * groups + threadIdx.x];
                tq += f_sq[sl * groups + threadIdx.x];
            }
            const double n = (double)HW * cpg;
            const double m1 = ts / n;                                            // mean of x - K_g
            double var = tq / n - m1 * m1;
            if (var < 0.0) var = 0.0;
            const double mean = (double)LbType<T>::to_f(base[threadIdx.x * cpg]) + m1;
            stats[(long long)b * groups + threadIdx.x] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
        }
        if (threadIdx.x == 0) counter[b] = 0;       // ready for the next launch that shares this workspace
    }
}

// pass 2: normalise, affine, optional SiLU.  Scale / shift of the thread's 8 channels live in registers.
template <typename T>
__global__ void __launch_bounds__(kThreads)
gn_apply_kernel(const T* __restrict__ x, long long ld, int C, int HW, int groups,
                const float2* __restrict__ stats, const T* __restrict__ gamma,
                const T* __restrict__ beta, int do_silu, T* __restrict__ out, long long ldo,
                int rows_per_block) {
    using L = LbType<T>;
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.y;
    const int VP = C >> 3;
    const int cpg = C / groups;
    const int RL = VP <= kThreads ? kThreads / VP : 1;
    const int row0 = blockIdx.x * rows_per_block;
    const int row1 = min(HW, row0 + rows_per_block);
    for (int cv0 = 0; cv0 < VP; cv0 += kThreads) {
        const int cv = cv0 + (VP <= kThreads ? (int)threadIdx.x % VP : (int)threadIdx.x);
        const int rl = VP <= kThreads ? (int)threadIdx.x / VP : 0;
        if (cv >= VP || rl >= RL) continue;
        float sc[8], sh[8];
        {
            const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gamma + 8 * cv));
            const uint4 bv = __ldg(reinterpret_cast<const uint4*>(beta + 8 * cv));
            const T* gh = reinterpret_cast<const T*>(&gv);
            const T* bh = reinterpret_cast<const T*>(&bv);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float2 st = stats[(long long)b * groups + (8 * cv + j) / cpg];     // (mean, rstd)
                sc[j] = st.y * L::to_f(gh[j]);
                sh[j] = L::to_f(bh[j]) - st.x * sc[j];
            }
        }
        const T* col = x + ((long long)b * HW) * ld + 8 * cv;
        T* ocol = out + ((long long)b * HW) * ldo + 8 * cv;
#pragma unroll 4
        for (int r = row0 + rl; r < row1; r += RL) {
            const uint4 v = *reinterpret_cast<const uint4*>(col + (long long)r * ld);
            const auto* h = reinterpret_cast<const typename L::T2*>(&v);
            uint4 o;
            auto* oh = reinterpret_cast<typename L::T2*>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = L::to_f2(h[j]);
                float y0 = L::round(fmaf(f.x, sc[2 * j], sh[2 * j]));
                float y1 = L::round(fmaf(f.y, sc[2 * j + 1], sh[2 * j + 1]));
                if (do_silu) {
                    y0 = silu_f(y0);
                    y1 = silu_f(y1);
                }
                oh[j] = L::from_f2(y0, y1);
            }
            *reinterpret_cast<uint4*>(ocol + (long long)r * ldo) = o;
        }
    }
}

// ---- LayerNorm: one warp per row, row held in registers -------------------------------------
template <int MAXV>
__global__ void __launch_bounds__(kThreads)
ln_kernel(const __half* __restrict__ x, long long ld, long long rows, int C, const __half* __restrict__ gamma,
          const __half* __restrict__ beta, float eps, __half* __restrict__ out, long long ldo) {
    pdl_launch_dependents();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (kThreads / 32) + warp;
    if (row >= rows) return;
    const int vecs = C >> 3;
    uint4 v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < vecs) {
            v[i] = *reinterpret_cast<const uint4*>(x + row * ld + vi * 8);
            const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                s += f.x + f.y;
            }
        }
    }
    s = lb_warp_sum(s);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < vecs) {
            const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                q = fmaf(f.x - mean, f.x - mean, q);
                q = fmaf(f.y - mean, f.y - mean, q);
            }
        }
    }
    q = lb_warp_sum(q);
    const float rstd = rsqrtf(q / (float)C + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < vecs) {
            const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
            const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gamma + vi * 8));
            const uint4 bv = __ldg(reinterpret_cast<const uint4*>(beta + vi * 8));
            const __half2* gh = reinterpret_cast<const __half2*>(&gv);
            const __half2* bh = reinterpret_cast<const __half2*>(&bv);
            uint4 o;
            __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                const float2 g = __half22float2(gh[j]);
                const float2 bb = __half22float2(bh[j]);
                oh[j] = __floats2half2_rn(fmaf((f.x - mean) * rstd, g.x, bb.x), fmaf((f.y - mean) * rstd, g.y, bb.y));
            }
            *reinterpret_cast<uint4*>(out + row * ldo + vi * 8) = o;
        }
    }
}

}  // namespace

// row chunks of pass 1: a function of HW only (batch-invariant results)
static int gn_rows_per_chunk(int HW) {
    int rpc = (int)lb_ceil_div(HW, 296);      // at most 296 chunks (2 per SM) per batch element ...
    if (rpc < 16) rpc = 16;                   // ... of at least 16 rows, so mid-size activations still fill the SMs
    if (rpc > HW) rpc = HW;
    return rpc;
}
static int gn_chunks(int HW) { return (int)lb_ceil_div(HW, gn_rows_per_chunk(HW)); }

// workspace: [kGnMaxBatch] int counters (must start zeroed; every launch leaves them zeroed -- they sit at a fixed
// offset so one zero-filled buffer can be shared by calls of different shapes) | [B][groups] float2 stats |
// [B][chunks][groups] float2 partials
constexpr int kGnMaxBatch = 64;
extern "C" size_t lb_groupnorm_workspace_bytes(lb_ctx* ctx, int B, int HW, int groups) {
    if (!ctx) return 0;
    return kGnMaxBatch * sizeof(int) + ((size_t)B * gn_chunks(HW) * groups + (size_t)B * groups) * sizeof(float2);
}

template <typename T>
static int groupnorm_launch(lb_ctx* ctx, const void* x, int64_t ld, int B, int HW, int C, int groups,
                            const void* gamma, const void* beta, float eps, int silu, void* out, int64_t ldo,
                            void* workspace, void* stream) {
    LB_REQUIRE(ctx && x && gamma && beta && out && workspace, "lb_groupnorm: null argument");
    LB_REQUIRE(groups >= 1 && groups <= 64 && C % groups == 0, "lb_groupnorm: C=%d groups=%d", C, groups);
    LB_REQUIRE(C % 8 == 0 && C <= kMaxC, "lb_groupnorm: C must be a multiple of 8 and <= %d (got %d)", kMaxC, C);
    LB_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && lb_aligned16(x) && lb_aligned16(out) && lb_aligned16(gamma) &&
                   lb_aligned16(beta), "lb_groupnorm: alignment");
    const int rpc = gn_rows_per_chunk(HW);
    const int chunks = gn_chunks(HW);
    LB_REQUIRE(B >= 1 && B <= kGnMaxBatch, "lb_groupnorm: batch %d > %d", B, kGnMaxBatch);
    int* counter = static_cast<int*>(workspace);
    float2* stats = reinterpret_cast<float2*>(counter + kGnMaxBatch);
    float2* partial = stats + (size_t)B * groups;
    cudaStream_t st = lb_stream(stream);
    lb_launch_pdl(gn_partial_kernel<T>, dim3(chunks, B), kThreads, 0, st, (const T*)x, ld, C, HW, groups, rpc, eps,
                  partial, stats, counter);
    LB_LAUNCH_CHECK();
    // apply: ~6 blocks per SM over the whole batch, at least 4 rows per row lane
    const int VP = C / 8;
    const int RL = VP <= kThreads ? kThreads / VP : 1;
    int blocks = (6 * ctx->sm_count + B - 1) / B;
    int rpb = (int)lb_ceil_div(HW, blocks);
    if (rpb < 4 * RL) rpb = 4 * RL;
    if (rpb > HW) rpb = HW;
    blocks = (int)lb_ceil_div(HW, rpb);
    lb_launch_pdl(gn_apply_kernel<T>, dim3(blocks, B), kThreads, 0, st, (const T*)x, ld, C, HW, groups,
                  (const float2*)stats, (const T*)gamma, (const T*)beta, silu, (T*)out, ldo, rpb);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_groupnorm(lb_ctx* ctx, const void* x, int64_t ld, int B, int HW, int C, int groups,
                            const void* gamma, const void* beta, float eps, int silu, void* out, int64_t ldo,
                            void* workspace, void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_groupnorm: unknown dtype %d", dtype);
    return dtype == LB_DTYPE_BF16
               ? groupnorm_launch<__nv_bfloat16>(ctx, x, ld, B, HW, C, groups, gamma, beta, eps, silu, out, ldo,
                                                 workspace, stream)
               : groupnorm_launch<__half>(ctx, x, ld, B, HW, C, groups, gamma, beta, eps, silu, out, ldo, workspace,
                                          stream);
}

extern "C" int lb_layernorm(lb_ctx* ctx, const void* x, int64_t ld, int64_t rows, int C, const void* gamma,
                            const void* beta, float eps, void* out, int64_t ldo, void* stream) {
    LB_REQUIRE(ctx && x && gamma && beta && out, "lb_layernorm: null argument");
    LB_REQUIRE(C % 8 == 0 && C <= 2048, "lb_layernorm: C must be a multiple of 8 and <= 2048 (got %d)", C);
    LB_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && lb_aligned16(x) && lb_aligned16(out) && lb_aligned16(gamma) &&
                   lb_aligned16(beta), "lb_layernorm: alignment");
    if (rows == 0) return 0;
    const unsigned grid = (unsigned)lb_ceil_div(rows, kThreads / 32);
    cudaStream_t st = lb_stream(stream);
    const int vecs = C / 8;
    if (vecs <= 64)
        lb_launch_pdl(ln_kernel<2>, grid, kThreads, 0, st, (const __half*)x, ld, rows, C, (const __half*)gamma,
                                                (const __half*)beta, eps, (__half*)out, ldo);
    else if (vecs <= 160)
        lb_launch_pdl(ln_kernel<5>, grid, kThreads, 0, st, (const __half*)x, ld, rows, C, (const __half*)gamma,
                                                (const __half*)beta, eps, (__half*)out, ldo);
    else
        lb_launch_pdl(ln_kernel<8>, grid, kThreads, 0, st, (const __half*)x, ld, rows, C, (const __half*)gamma,
                                                (const __half*)beta, eps, (__half*)out, ldo);
    LB_LAUNCH_CHECK();
    return 0;
}
