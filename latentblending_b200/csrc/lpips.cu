// lpips.cu -- SURVEY section 8(f) rows #2 and #3 on the device:
//
//   #2  LPIPS-AlexNet branch-placement metric (latentblending/blending_engine.py:744-758, lpips==0.1.4 un-vendored):
//       the five AlexNet convolutions run on the wgmma GEMM (lb_gemm with the ReLU epilogue) over patch matrices
//       produced here -- conv1 straight from the uint8 frame with the [-1,1] + ScalingLayer arithmetic fused
//       (the reference round-trips every frame through PIL and a host->device copy, :750-755) -- plus the 3x3/2
//       max-pools and the fused "unit-normalise, squared difference, 1x1 lin, spatial mean" tap reduction.
//   #3  the linear frame fill of write_movie_transition (blending_engine.py:684-706 -> utils.py:105-178):
//       out[t] = uint8( fl32(w0[t]*a) + fl32(w1[t]*b) ) for a list of (left frame, weights) -- numpy's float32
//       arithmetic (no FMA contraction) and its truncating uint8 cast.
// All HBM-bound: 128-bit accesses, grid sized in multiples of the SM count.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

unsigned grid_for(long long work_items, int sm) {
    long long g = lb_ceil_div(work_items, kThreads);
    const long long cap = (long long)sm * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (unsigned)g;
}

// ---- conv1 patch matrix from a uint8 HWC frame -------------------------------------------------------
// row = output pixel (oy, ox); column j = (ky*k + kx)*3 + c for j < 3*k*k, zero for the padding columns up to Kp.
// value = ((2*u/255 - 1) - shift[c]) / scale[c]   (blending_engine.py:750-755 + lpips ScalingLayer), 0 outside the frame
// (the convolution zero-pads the SCALED input).
__global__ void __launch_bounds__(kThreads)
lpips_im2col_u8_kernel(const uint8_t* __restrict__ img, int H, int W, int k, int stride, int pad, int Ho, int Wo, int Kp,
                       float sh0, float sh1, float sh2, float sc0, float sc1, float sc2, __half* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const int vecs = Kp >> 3;
    const long long total = (long long)Ho * Wo * vecs;
    const int kk3 = 3 * k * k;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int v = (int)(i % vecs);
        const long long r = i / vecs;
        const int ox = (int)(r % Wo), oy = (int)(r / Wo);
        uint4 o;
        __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int j = v * 8 + e;
            float val = 0.f;
            if (j < kk3) {
                const int c = j % 3, t = j / 3;
                const int kx = t % k, ky = t / k;
                const int y = oy * stride - pad + ky, x = ox * stride - pad + kx;
                if (y >= 0 && y < H && x >= 0 && x < W) {
                    const float u = (float)img[((long long)y * W + x) * 3 + c];
                    const float s = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, u), 255.0f), 1.0f);
                    const float sh = c == 0 ? sh0 : c == 1 ? sh1 : sh2;
                    const float sc = c == 0 ? sc0 : c == 1 ? sc1 : sc2;
                    val = __fdiv_rn(__fsub_rn(s, sh), sc);
                }
            }
            oh[e] = __float2half_rn(val);
        }
        reinterpret_cast<uint4*>(out)[i] = o;
    }
}

// ---- generic NHWC patch matrix: out[(oy,ox)][(ky*k+kx)*C + c] = x[oy*s-p+ky][ox*s-p+kx][c] (zero padded) --------
__global__ void __launch_bounds__(kThreads)
im2col_nhwc_kernel(const __half* __restrict__ x, long long ld, int H, int W, int C, int k, int stride, int pad, int Ho,
                   int Wo, __half* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const int cv = C >> 3;
    const int taps = k * k;
    const long long total = (long long)Ho * Wo * taps * cv;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int c8 = (int)(i % cv);
        const long long q = i / cv;
        const int t = (int)(q % taps);
        const long long r = q / taps;
        const int ox = (int)(r % Wo), oy = (int)(r / Wo);
        const int kx = t % k, ky = t / k;
        const int y = oy * stride - pad + ky, xx = ox * stride - pad + kx;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (y >= 0 && y < H && xx >= 0 && xx < W)
            v = *reinterpret_cast<const uint4*>(x + ((long long)y * W + xx) * ld + c8 * 8);
        reinterpret_cast<uint4*>(out)[i] = v;
    }
}

// ---- MaxPool2d(3, stride 2), NHWC ---------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
maxpool3s2_kernel(const __half* __restrict__ x, long long ld, int H, int W, int C, int Ho, int Wo,
                  __half* __restrict__ out, long long ldo) {
    pdl_launch_dependents();
    pdl_wait();
    const int cv = C >> 3;
    const long long total = (long long)Ho * Wo * cv;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int c8 = (int)(i % cv);
        const long long r = i / cv;
        const int ox = (int)(r % Wo), oy = (int)(r / Wo);
        __half2 m[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = __float2half2_rn(-65504.0f);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int y = 2 * oy + ky, xx = 2 * ox + kx;
                if (y < H && xx < W) {
                    const uint4 v = *reinterpret_cast<const uint4*>(x + ((long long)y * W + xx) * ld + c8 * 8);
                    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
                    for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], h[j]);
                }
            }
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) oh[j] = m[j];
        *reinterpret_cast<uint4*>(out + r * ldo + c8 * 8) = o;
    }
}

// ---- one LPIPS tap: sum over pixels of  sum_c lin[c] * (a_c/(|a|+eps) - b_c/(|b|+eps))^2 ---------------------------
// One warp per pixel (row of the [rows, C] feature matrices), fp32 arithmetic on the fp16 features; a block writes ONE
// partial (fixed intra-block order), lpips_tap_final adds the partials in index order -> deterministic.
constexpr int kTapMaxPerLane = 16;      // C <= 32 * 16 = 512 channels
__global__ void __launch_bounds__(kThreads)
lpips_tap_kernel(const __half* __restrict__ fa, const __half* __restrict__ fb, long long ld, long long rows, int C,
                 const float* __restrict__ lin, float* __restrict__ partial) {
    pdl_launch_dependents();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wpb = kThreads / 32;
    const int per = C / 64;                 // half2 pairs per lane (C is a multiple of 64)
    float acc = 0.f;
    for (long long r = (long long)blockIdx.x * wpb + warp; r < rows; r += (long long)gridDim.x * wpb) {
        float2 a[kTapMaxPerLane / 2], b[kTapMaxPerLane / 2];
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int i = 0; i < kTapMaxPerLane / 2; ++i) {
            if (i < per) {
                a[i] = __half22float2(*reinterpret_cast<const __half2*>(fa + r * ld + 2 * lane + 64 * i));
                b[i] = __half22float2(*reinterpret_cast<const __half2*>(fb + r * ld + 2 * lane + 64 * i));
                sa += a[i].x * a[i].x + a[i].y * a[i].y;
                sb += b[i].x * b[i].x + b[i].y * b[i].y;
            }
        }
        sa = lb_warp_sum(sa);
        sb = lb_warp_sum(sb);
        const float ia = 1.0f / (sqrtf(sa) + 1e-10f), ib = 1.0f / (sqrtf(sb) + 1e-10f);
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < kTapMaxPerLane / 2; ++i) {
            if (i < per) {
                const float2 l = *reinterpret_cast<const float2*>(lin + 2 * lane + 64 * i);
                const float dx = a[i].x * ia - b[i].x * ib, dy = a[i].y * ia - b[i].y * ib;
                d += l.x * dx * dx + l.y * dy * dy;
            }
        }
        acc += lb_warp_sum(d);
    }
    __shared__ float s[kThreads / 32];
    if (lane == 0) s[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < wpb; ++w) t += s[w];
        partial[blockIdx.x] = t;
    }
}

__global__ void lpips_tap_final_kernel(const float* __restrict__ partial, int n_partial, float inv_rows, int accumulate,
                                       float* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < n_partial; ++i) t += partial[i];
        const float v = t * inv_rows;
        out[0] = accumulate ? out[0] + v : v;
    }
}

// ---- frame fill: out[t] = trunc_u8( fl32(w0[t]*frames[left[t]]) + fl32(w1[t]*frames[left[t]+1]) ) -----------------------
__global__ void __launch_bounds__(kThreads)
frames_lerp_u8_kernel(const uint8_t* __restrict__ frames, long long n, const int* __restrict__ left,
                      const float* __restrict__ w0, const float* __restrict__ w1, int T, uint8_t* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const long long nv = n >> 4;
    const long long total = nv * T;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int t = (int)(i / nv);
        const long long v = i % nv;
        const int l = left[t];
        const float a0 = w0[t], a1 = w1[t];
        const uint4 va = reinterpret_cast<const uint4*>(frames + (long long)l * n)[v];
        uint4 vo = va;
        if (a1 != 0.0f) {
            const uint4 vb = reinterpret_cast<const uint4*>(frames + (long long)(l + 1) * n)[v];
            const uint8_t* pa = reinterpret_cast<const uint8_t*>(&va);
            const uint8_t* pb = reinterpret_cast<const uint8_t*>(&vb);
            uint8_t* po = reinterpret_cast<uint8_t*>(&vo);
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                const float r = __fadd_rn(__fmul_rn(a0, (float)pa[e]), __fmul_rn(a1, (float)pb[e]));
                po[e] = (uint8_t)(int)r;         // numpy .astype(uint8): truncation (values are within [0, 255])
            }
        }
        reinterpret_cast<uint4*>(out + (long long)t * n)[v] = vo;
    }
}

}  // namespace

extern "C" int lb_lpips_im2col_u8(lb_ctx* ctx, const void* frame_u8, int H, int W, int k, int stride, int pad,
                                  const float* shift3, const float* scale3, void* out, int64_t out_cols, void* stream) {
    LB_REQUIRE(ctx && frame_u8 && out && shift3 && scale3, "lb_lpips_im2col_u8: null argument");
    LB_REQUIRE(k >= 1 && stride >= 1 && pad >= 0 && H + 2 * pad >= k && W + 2 * pad >= k, "lb_lpips_im2col_u8: bad geometry");
    LB_REQUIRE(out_cols % 8 == 0 && out_cols >= 3 * k * k && lb_aligned16(out), "lb_lpips_im2col_u8: out_cols must be a "
               "multiple of 8 and >= 3*k*k, out 16B aligned");
    const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    lb_launch_pdl(lpips_im2col_u8_kernel, grid_for((long long)Ho * Wo * (out_cols / 8), ctx->sm_count), kThreads, 0,
                  lb_stream(stream), (const uint8_t*)frame_u8, H, W, k, stride, pad, Ho, Wo, (int)out_cols, shift3[0],
                  shift3[1], shift3[2], scale3[0], scale3[1], scale3[2], (__half*)out);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_im2col(lb_ctx* ctx, const void* x, int64_t ld, int H, int W, int C, int k, int stride, int pad,
                         void* out, void* stream) {
    LB_REQUIRE(ctx && x && out, "lb_im2col: null argument");
    LB_REQUIRE(C % 8 == 0 && ld % 8 == 0 && lb_aligned16(x) && lb_aligned16(out), "lb_im2col: C / stride multiples of 8, "
               "16B aligned bases");
    LB_REQUIRE(k >= 1 && stride >= 1 && pad >= 0 && H + 2 * pad >= k && W + 2 * pad >= k, "lb_im2col: bad geometry");
    const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    lb_launch_pdl(im2col_nhwc_kernel, grid_for((long long)Ho * Wo * k * k * (C / 8), ctx->sm_count), kThreads, 0,
                  lb_stream(stream), (const __half*)x, (long long)ld, H, W, C, k, stride, pad, Ho, Wo, (__half*)out);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_maxpool3s2(lb_ctx* ctx, const void* x, int64_t ld, int H, int W, int C, void* out, int64_t ldo,
                             void* stream) {
    LB_REQUIRE(ctx && x && out, "lb_maxpool3s2: null argument");
    LB_REQUIRE(C % 8 == 0 && ld % 8 == 0 && ldo % 8 == 0 && lb_aligned16(x) && lb_aligned16(out) && H >= 3 && W >= 3,
               "lb_maxpool3s2: C / strides multiples of 8, 16B aligned bases, H, W >= 3");
    const int Ho = (H - 3) / 2 + 1, Wo = (W - 3) / 2 + 1;
    lb_launch_pdl(maxpool3s2_kernel, grid_for((long long)Ho * Wo * (C / 8), ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const __half*)x, (long long)ld, H, W, C, Ho, Wo, (__half*)out, (long long)ldo);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t lb_lpips_tap_workspace_bytes(lb_ctx* ctx) { return ctx ? (size_t)ctx->sm_count * 8 * sizeof(float) : 0; }

extern "C" int lb_lpips_tap(lb_ctx* ctx, const void* feat_a, const void* feat_b, int64_t ld, int64_t rows, int C,
                            const float* lin_w, int accumulate, float* out_scalar, void* workspace, void* stream) {
    LB_REQUIRE(ctx && feat_a && feat_b && lin_w && out_scalar && workspace, "lb_lpips_tap: null argument");
    LB_REQUIRE(C % 64 == 0 && C <= 32 * kTapMaxPerLane && ld % 2 == 0 && rows >= 1, "lb_lpips_tap: C must be a multiple of "
               "64 and <= 512 (got %d)", C);
    long long blocks = lb_ceil_div(rows, kThreads / 32);
    const long long cap = (long long)ctx->sm_count * 8;
    if (blocks > cap) blocks = cap;
    lb_launch_pdl(lpips_tap_kernel, (unsigned)blocks, kThreads, 0, lb_stream(stream), (const __half*)feat_a,
                  (const __half*)feat_b, (long long)ld, (long long)rows, C, lin_w, (float*)workspace);
    LB_LAUNCH_CHECK();
    lb_launch_pdl(lpips_tap_final_kernel, 1, 32, 0, lb_stream(stream), (const float*)workspace, (int)blocks,
                  1.0f / (float)rows, accumulate, out_scalar);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_frames_lerp_u8(lb_ctx* ctx, const void* frames_u8, int64_t n, const int* left_idx_dev,
                                 const float* w0_dev, const float* w1_dev, int T, void* out_u8, void* stream) {
    LB_REQUIRE(ctx && frames_u8 && left_idx_dev && w0_dev && w1_dev && out_u8, "lb_frames_lerp_u8: null argument");
    LB_REQUIRE(n % 16 == 0 && lb_aligned16(frames_u8) && lb_aligned16(out_u8) && T >= 1,
               "lb_frames_lerp_u8: frame size must be a multiple of 16 bytes, bases 16B aligned");
    lb_launch_pdl(frames_lerp_u8_kernel, grid_for((n / 16) * T, ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const uint8_t*)frames_u8, (long long)n, left_idx_dev, w0_dev, w1_dev, T, (uint8_t*)out_u8);
    LB_LAUNCH_CHECK();
    return 0;
}
