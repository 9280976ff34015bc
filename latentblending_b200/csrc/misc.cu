// misc.cu -- the small / memory-bound pieces of the UNet forward that are not GEMM-shaped:
//   K3  timestep + added-condition embedding inputs (sinusoids) and the small-M linears
//       (time_embedding, add_embedding, all resnet time_emb_proj in one batched launch)
//   K2  conv_in  (4 -> C0, 3x3, NCHW latent in, NHWC out)
//       nearest upsample (2x, or 2x cropped by one row / column), stride-2 im2col (the two Downsample2D convs then run as plain GEMMs)
//       the T2I-Adapter's pixel unshuffle and ceil-mode 2x2 average pool, and its in-place state add
// Replace pieces of pipe.unet(...) (call site latentblending/diffusers_holder.py:336-344;
// diffusers 0.25.0 embeddings.py / resnet.py / unet_2d_condition.py).
#include "common.cuh"

#include <type_traits>

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

// ---- embedding inputs ---------------------------------------------------------------------
// temb_in[b, :dim_t]            = [cos(t*f_i) | sin(t*f_i)],  f_i = exp(-ln(1e4) * i / (dim_t/2))
// add_in[b, :pooled]            = text_embeds[b]
// add_in[b, pooled + 6*j ...]   = sinusoid(time_ids[b, j], dim_a)   (flip_sin_to_cos: cos first)
// t_dev (optional): the timestep is read from device memory instead of the launch parameter, so that a CUDA graph of
// the whole UNet program can be replayed for any timestep (program.cu).
__global__ void embed_inputs_kernel(float t, const float* __restrict__ t_dev, const __half* __restrict__ text_embeds,
                                    const __half* __restrict__ time_ids,
                                    int B, int dim_t, int pooled, int dim_a, __half* __restrict__ temb_in,
                                    __half* __restrict__ add_in) {
    pdl_launch_dependents();
    pdl_wait();
    if (t_dev != nullptr) t = *t_dev;
    const int b = blockIdx.x;
    const int half_t = dim_t / 2, half_a = dim_a / 2;
    const int add_w = pooled + 6 * dim_a;
    for (int i = threadIdx.x; i < dim_t; i += blockDim.x) {
        const int k = i % half_t;
        const float f = expf(-9.210340371976184f * (float)k / (float)half_t);
        const float a = t * f;
        temb_in[(long long)b * dim_t + i] = __float2half_rn(i < half_t ? cosf(a) : sinf(a));
    }
    for (int i = threadIdx.x; i < add_w; i += blockDim.x) {
        __half v;
        if (i < pooled) {
            v = text_embeds[(long long)b * pooled + i];
        } else {
            const int j = (i - pooled) / dim_a, k = (i - pooled) % dim_a;
            const int kk = k % half_a;
            const float f = expf(-9.210340371976184f * (float)kk / (float)half_a);
            const float a = __half2float(time_ids[b * 6 + j]) * f;
            v = __float2half_rn(k < half_a ? cosf(a) : sinf(a));
        }
        add_in[(long long)b * add_w + i] = v;
    }
}

// ---- small-M linear: out[m,n] = act_out( x_act[m,:] . w[n,:] + bias[n] ) (+ addend[m,n]) -------------
// One warp per output column; M <= 16 rows; weight-read bound (each weight row is read once).
template <int MAXM>
__global__ void __launch_bounds__(kThreads)
linear_small_kernel(const __half* __restrict__ x, long long ldx, int M, int K, const __half* __restrict__ w,
                    long long ldw, const __half* __restrict__ bias, const __half* __restrict__ addend,
                    long long ldadd, int act_in, int act_out, __half* __restrict__ out, long long ldo, int N) {
    pdl_launch_dependents();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = blockIdx.x * (kThreads / 32) + warp;
    if (n >= N) return;
    float acc[MAXM];
#pragma unroll
    for (int m = 0; m < MAXM; ++m) acc[m] = 0.f;
    const int vecs = K >> 3;
    for (int v = lane; v < vecs; v += 32) {
        const uint4 wv = lb_ldg_stream(w + (long long)n * ldw + v * 8);
        const __half2* wh = reinterpret_cast<const __half2*>(&wv);
        float wf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(wh[j]);
            wf[2 * j] = f.x;
            wf[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int m = 0; m < MAXM; ++m) {
            if (m < M) {
                const uint4 xv = *reinterpret_cast<const uint4*>(x + (long long)m * ldx + v * 8);
                const __half2* xh = reinterpret_cast<const __half2*>(&xv);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float2 f = __half22float2(xh[j]);
                    if (act_in) {
                        f.x = lb_round_h(silu_f(f.x));
                        f.y = lb_round_h(silu_f(f.y));
                    }
                    acc[m] = fmaf(f.x, wf[2 * j], acc[m]);
                    acc[m] = fmaf(f.y, wf[2 * j + 1], acc[m]);
                }
            }
        }
    }
#pragma unroll
    for (int m = 0; m < MAXM; ++m) acc[m] = lb_warp_sum(acc[m]);
    if (lane == 0) {
        const float bn = bias ? __half2float(bias[n]) : 0.f;
        for (int m = 0; m < M; ++m) {
            float y = lb_round_h(acc[m] + bn);
            if (act_out) y = lb_round_h(silu_f(y));
            if (addend) y = lb_round_h(y + __half2float(addend[(long long)m * ldadd + n]));
            out[(long long)m * ldo + n] = __float2half_rn(y);
        }
    }
}

// ---- conv_in: NCHW [B,Cin<=8,H,W] -> NHWC [B*H*W, Cout], 3x3 pad 1 -------------------------------
// weights packed [ky][kx][cin][Cout] fp16 (bf16 in the bf16 variant) so a lane reads 8 consecutive output channels.
// kTiny (lb_conv_in act 1, fp16): the tiny VAE decoder's input stage -- every input v is clamped to
// h(h(tanh(h(h(v * in_scale) / 3))) * 3) (h: fp16 rounding, at the reference's points), and ReLU follows the conv.
__device__ __forceinline__ float tiny_vae_input(float v, float in_scale) {
    const float z = lb_round_h(v * in_scale);
    return lb_round_h(lb_round_h(tanhf(lb_round_h(z / 3.0f))) * 3.0f);
}

// kAdd (lb_conv_in_add, fp16): out = h(h(conv + bias) + addend[pix mod H*W]) -- a ControlNet's
// ``conv_in(x) + controlnet_cond_embedding(image)`` with one embedding row per pixel shared by every batch row.
template <typename T, bool kTiny, bool kAdd = false>
__device__ __forceinline__ void conv_in_body(const T* __restrict__ x, int B, int Cin, int H, int W,
                                             const T* __restrict__ wp, const T* __restrict__ bias, int Cout,
                                             T* __restrict__ out, long long ldo, float in_scale,
                                             const T* __restrict__ addend = nullptr, long long ld_add = 0) {
    using L = LbType<T>;
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ __half s_w_raw[];
    T* s_w = reinterpret_cast<T*>(s_w_raw);   // [9*Cin][Cout] (T is 2 bytes, like __half)
    const int wn = 9 * Cin * Cout;
    for (int i = threadIdx.x; i < wn; i += kThreads) s_w[i] = wp[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long npix = (long long)B * H * W;
    const int groups = Cout >> 3;
    for (long long pix = (long long)blockIdx.x * (kThreads / 32) + warp; pix < npix;
         pix += (long long)gridDim.x * (kThreads / 32)) {
        const int xw = (int)(pix % W), yh = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
        for (int g = lane; g < groups; g += 32) {
            float acc[8];
            {
                const uint4 bv = *reinterpret_cast<const uint4*>(bias + g * 8);
                const auto* bh = reinterpret_cast<const typename L::T2*>(&bv);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = L::to_f2(bh[j]);
                    acc[2 * j] = f.x;
                    acc[2 * j + 1] = f.y;
                }
            }
            for (int ky = 0; ky < 3; ++ky) {
                const int yy = yh + ky - 1;
                if (yy < 0 || yy >= H) continue;
                for (int kx = 0; kx < 3; ++kx) {
                    const int xx = xw + kx - 1;
                    if (xx < 0 || xx >= W) continue;
                    for (int c = 0; c < Cin; ++c) {
                        float xv = L::to_f(x[(((long long)b * Cin + c) * H + yy) * W + xx]);
                        if constexpr (kTiny) xv = tiny_vae_input(xv, in_scale);
                        const uint4 wv = *reinterpret_cast<const uint4*>(s_w + ((ky * 3 + kx) * Cin + c) * Cout + g * 8);
                        const auto* wh = reinterpret_cast<const typename L::T2*>(&wv);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float2 f = L::to_f2(wh[j]);
                            acc[2 * j] = fmaf(xv, f.x, acc[2 * j]);
                            acc[2 * j + 1] = fmaf(xv, f.y, acc[2 * j + 1]);
                        }
                    }
                }
            }
            if constexpr (kTiny) {
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j], 0.f);
            }
            if constexpr (kAdd) {
                const uint4 av = *reinterpret_cast<const uint4*>(addend + (pix % ((long long)H * W)) * ld_add + g * 8);
                const auto* ah = reinterpret_cast<const typename L::T2*>(&av);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = L::to_f2(ah[j]);
                    acc[2 * j] = L::round(acc[2 * j]) + f.x;
                    acc[2 * j + 1] = L::round(acc[2 * j + 1]) + f.y;
                }
            }
            uint4 o;
            auto* oh = reinterpret_cast<typename L::T2*>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) oh[j] = L::from_f2(acc[2 * j], acc[2 * j + 1]);
            *reinterpret_cast<uint4*>(out + pix * ldo + g * 8) = o;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
conv_in_kernel(const T* __restrict__ x, int B, int Cin, int H, int W, const T* __restrict__ wp,
               const T* __restrict__ bias, int Cout, T* __restrict__ out, long long ldo) {
    conv_in_body<T, false>(x, B, Cin, H, W, wp, bias, Cout, out, ldo, 1.0f);
}

__global__ void __launch_bounds__(kThreads)
conv_in_tiny_kernel(const __half* __restrict__ x, int B, int Cin, int H, int W, const __half* __restrict__ wp,
                    const __half* __restrict__ bias, int Cout, __half* __restrict__ out, long long ldo, float in_scale) {
    conv_in_body<__half, true>(x, B, Cin, H, W, wp, bias, Cout, out, ldo, in_scale);
}

__global__ void __launch_bounds__(kThreads)
conv_in_add_kernel(const __half* __restrict__ x, int B, int Cin, int H, int W, const __half* __restrict__ wp,
                   const __half* __restrict__ bias, int Cout, __half* __restrict__ out, long long ldo,
                   const __half* __restrict__ addend, long long ld_add) {
    conv_in_body<__half, false, true>(x, B, Cin, H, W, wp, bias, Cout, out, ldo, 1.0f, addend, ld_add);
}

// ---- nearest upsample to Ho x Wo (Ho in {2H-1, 2H}, Wo in {2W-1, 2W}), NHWC ------------------------------------
// Nearest 2x cropped to Ho x Wo: output (yo, xo) reads input (yo >> 1, xo >> 1).  With H = ceil(Ho / 2) this is
// exactly torch's nearest index min(floor(yo * (float)H / Ho), H - 1), so F.interpolate(size=...) needs no
// floating-point index arithmetic here.
__global__ void __launch_bounds__(kThreads)
upsample_nearest_kernel(const __half* __restrict__ x, long long ld, int B, int H, int W, int C, __half* __restrict__ out,
                        long long ldo, int Ho, int Wo) {
    pdl_launch_dependents();
    pdl_wait();
    const int vecs = C >> 3;
    const long long total = (long long)B * Ho * Wo * vecs;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int v = (int)(i % vecs);
        const long long opix = i / vecs;
        const int xo = (int)(opix % Wo), yo = (int)((opix / Wo) % Ho), b = (int)(opix / ((long long)Wo * Ho));
        const long long ipix = ((long long)b * H + (yo >> 1)) * W + (xo >> 1);
        *reinterpret_cast<uint4*>(out + opix * ldo + v * 8) = *reinterpret_cast<const uint4*>(x + ipix * ld + v * 8);
    }
}

// ---- im2col for the 3x3 stride-2 downsample convs: out[B*Ho*Wo, 9*C], K order (ky,kx,c) ------
// kPadLo = 1: zero padding 1 on every side (the UNet's Downsample2D), Ho = floor((H + 2 - 3)/2) + 1.
// kPadLo = 0: F.pad(x, (0, 1, 0, 1)) then no padding (the VAE encoder's Downsample2D(padding=0)),
//             Ho = floor((H + 1 - 3)/2) + 1.  The kernel copies 16-byte channel vectors: fp16 and bf16 alike.
template <int kPadLo>
__global__ void __launch_bounds__(kThreads)
im2col_s2_kernel(const __half* __restrict__ x, long long ld, int B, int H, int W, int C, __half* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const int Ho = kPadLo ? (H + 1) / 2 : (H - 2) / 2 + 1, Wo = kPadLo ? (W + 1) / 2 : (W - 2) / 2 + 1;
    const int vecs = C >> 3;
    const long long total = (long long)B * Ho * Wo * 9 * vecs;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int v = (int)(i % vecs);
        const int tap = (int)((i / vecs) % 9);
        const long long opix = i / ((long long)vecs * 9);
        const int xo = (int)(opix % Wo), yo = (int)((opix / Wo) % Ho), b = (int)(opix / ((long long)Wo * Ho));
        const int yy = 2 * yo + tap / 3 - kPadLo, xx = 2 * xo + tap % 3 - kPadLo;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (yy >= 0 && yy < H && xx >= 0 && xx < W)
            val = *reinterpret_cast<const uint4*>(x + (((long long)b * H + yy) * W + xx) * ld + v * 8);
        *reinterpret_cast<uint4*>(out + opix * (9LL * C) + (long long)tap * C + v * 8) = val;
    }
}

// ---- T2I-Adapter pieces -------------------------------------------------------------------------------------------
// add_rows_bcast: dst[b*rows + r, :C] += src[r, :C] for every batch row b: the adapter's per-image state added in
// place to a skip (or the mid output) of every CFG half / lockstep job.  fp32 add, one rounding: torch's fp16 ``+=``.
__global__ void __launch_bounds__(kThreads)
add_rows_bcast_kernel(__half* __restrict__ dst, long long ld_dst, const __half* __restrict__ src, long long ld_src,
                      int B, long long rows, int C) {
    pdl_launch_dependents();
    pdl_wait();
    const int vecs = C >> 3;
    const long long total = (long long)B * rows * vecs;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int v = (int)(i % vecs);
        const long long row = i / vecs, r = row % rows;
        uint4* d = reinterpret_cast<uint4*>(dst + row * ld_dst + v * 8);
        uint4 a = *d;
        const uint4 s = *reinterpret_cast<const uint4*>(src + r * ld_src + v * 8);
        __half2* ah = reinterpret_cast<__half2*>(&a);
        const __half2* sh = reinterpret_cast<const __half2*>(&s);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 x = __half22float2(ah[j]), y = __half22float2(sh[j]);
            ah[j] = __floats2half2_rn(x.x + y.x, x.y + y.y);
        }
        *d = a;
    }
}

// pixel_unshuffle_u8: uint8 image [H, W, Cimg] -> fp16 [(H/r)*(W/r), r*r*Cimg], fp16(float(u) / 255), columns in
// (i, j, c) order (i, j the offset inside the r x r block).  Row i of a block is r*Cimg consecutive image bytes, so
// each thread converts 8 consecutive bytes into one 16-byte store.  F.pixel_unshuffle's (c, i, j) order is the
// caller's weight permutation.
__global__ void __launch_bounds__(kThreads)
pixel_unshuffle_u8_kernel(const uint8_t* __restrict__ img, int H, int W, int Cimg, int r, __half* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const int Wo = W / r, seg = r * Cimg, K = seg * r, vecs = K >> 3;
    const long long total = (long long)(H / r) * Wo * vecs;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int v = (int)(i % vecs);
        const long long opix = i / vecs;
        const int xo = (int)(opix % Wo), yo = (int)(opix / Wo);
        const int col = v * 8, bi = col / seg, off = col % seg;
        const uint2 raw = *reinterpret_cast<const uint2*>(img + ((long long)(yo * r + bi) * W + (long long)xo * r) * Cimg + off);
        const uint8_t* b = reinterpret_cast<const uint8_t*>(&raw);
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn((float)b[2 * j] / 255.0f, (float)b[2 * j + 1] / 255.0f);
        *reinterpret_cast<uint4*>(out + opix * K + col) = o;
    }
}

// avgpool2_ceil: NHWC AvgPool2d(2, stride 2, ceil_mode=True, padding 0): Ho = ceil(H/2); a window hanging over the
// bottom / right edge is clipped and divided by its in-bounds count.  fp32 sum in row-major window order, then the
// division, one rounding: torch's avg_pool2d on fp16.
__global__ void __launch_bounds__(kThreads)
avgpool2_ceil_kernel(const __half* __restrict__ x, long long ld, int H, int W, int C, __half* __restrict__ out,
                     long long ldo) {
    pdl_launch_dependents();
    pdl_wait();
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2, vecs = C >> 3;
    const long long total = (long long)Ho * Wo * vecs;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int v = (int)(i % vecs);
        const long long opix = i / vecs;
        const int xo = (int)(opix % Wo), yo = (int)(opix / Wo);
        const int y1 = min(2 * yo + 2, H), x1 = min(2 * xo + 2, W);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int y = 2 * yo; y < y1; ++y)
            for (int xx = 2 * xo; xx < x1; ++xx) {
                const uint4 q = *reinterpret_cast<const uint4*>(x + ((long long)y * W + xx) * ld + v * 8);
                const __half2* qh = reinterpret_cast<const __half2*>(&q);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(qh[j]);
                    acc[2 * j] += f.x;
                    acc[2 * j + 1] += f.y;
                }
            }
        const float cnt = (float)((y1 - 2 * yo) * (x1 - 2 * xo));
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(acc[2 * j] / cnt, acc[2 * j + 1] / cnt);
        *reinterpret_cast<uint4*>(out + opix * ldo + v * 8) = o;
    }
}

unsigned grid_for(long long work_items, int sm) {
    long long g = lb_ceil_div(work_items, kThreads);
    const long long cap = (long long)sm * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (unsigned)g;
}

}  // namespace

// internal: t from device memory when t_dev != NULL (graph replay), else the launch parameter
int lb_embed_inputs_src(lb_ctx* ctx, float t, const float* t_dev, const void* text_embeds, const void* time_ids, int B,
                        int dim_t, int pooled, int dim_a, void* temb_in, void* add_in, void* stream) {
    LB_REQUIRE(ctx && text_embeds && time_ids && temb_in && add_in, "lb_embed_inputs: null argument");
    LB_REQUIRE(dim_t % 2 == 0 && dim_a % 2 == 0 && B >= 1, "lb_embed_inputs: bad sizes");
    lb_launch_pdl(embed_inputs_kernel, B, kThreads, 0, lb_stream(stream), t, t_dev, (const __half*)text_embeds,
                  (const __half*)time_ids, B, dim_t, pooled, dim_a, (__half*)temb_in, (__half*)add_in);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_embed_inputs(lb_ctx* ctx, float t, const void* text_embeds, const void* time_ids, int B,
                               int dim_t, int pooled, int dim_a, void* temb_in, void* add_in, void* stream) {
    return lb_embed_inputs_src(ctx, t, nullptr, text_embeds, time_ids, B, dim_t, pooled, dim_a, temb_in, add_in, stream);
}

__global__ void set_scalar_kernel(float* dst, float v) {
    pdl_launch_dependents();
    pdl_wait();
    *dst = v;
}
int lb_set_scalar(float* dst_dev, float v, cudaStream_t st) {
    lb_launch_pdl(set_scalar_kernel, 1, 1, 0, st, dst_dev, v);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_linear_small(lb_ctx* ctx, const void* x, int64_t ldx, int M, int K, const void* w, int64_t ldw,
                               const void* bias, const void* addend, int64_t ldadd, int act_in, int act_out,
                               void* out, int64_t ldo, int N, void* stream) {
    LB_REQUIRE(ctx && x && w && out, "lb_linear_small: null argument");
    LB_REQUIRE(M >= 1 && M <= 16, "lb_linear_small: M must be in [1,16] (got %d)", M);
    LB_REQUIRE(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0 && lb_aligned16(x) && lb_aligned16(w),
               "lb_linear_small: K / strides must be multiples of 8 and bases 16B aligned");
    const unsigned grid = (unsigned)lb_ceil_div(N, kThreads / 32);
    cudaStream_t st = lb_stream(stream);
#define LB_LS(MM)                                                                                                    \
    lb_launch_pdl(linear_small_kernel<MM>, grid, kThreads, 0, st, (const __half*)x, ldx, M, K, (const __half*)w, ldw,            \
                                                       (const __half*)bias, (const __half*)addend, ldadd, act_in,     \
                                                       act_out, (__half*)out, ldo, N)
    if (M <= 2) LB_LS(2);
    else if (M <= 4) LB_LS(4);
    else if (M <= 8) LB_LS(8);
    else LB_LS(16);
#undef LB_LS
    LB_LAUNCH_CHECK();
    return 0;
}

// One launcher for both conv_in kernels; ``extra`` is the kernel's arguments after ldo.
template <typename T, auto kKernel, typename... Extra>
static int conv_in_launch(lb_ctx* ctx, const void* x_nchw, int B, int Cin, int H, int W, const void* w_packed,
                          const void* bias, int Cout, void* out, int64_t ldo, void* stream, Extra... extra) {
    LB_REQUIRE(ctx && x_nchw && w_packed && bias && out, "lb_conv_in: null argument");
    LB_REQUIRE(Cin >= 1 && Cin <= 8 && Cout % 8 == 0 && ldo % 8 == 0, "lb_conv_in: Cin<=8, Cout%%8==0 required");
    const int smem = 9 * Cin * Cout * 2;
    LB_REQUIRE(smem <= 96 * 1024, "lb_conv_in: weights do not fit shared memory");
    static bool attr = false;      // one flag per kernel (per instantiation)
    if (!attr) {
        LB_CHECK_CUDA(cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr = true;
    }
    const long long npix = (long long)B * H * W;
    unsigned grid = (unsigned)lb_ceil_div(npix, kThreads / 32);
    if (grid > (unsigned)ctx->sm_count * 4) grid = ctx->sm_count * 4;
    lb_launch_pdl(kKernel, grid, kThreads, smem, lb_stream(stream), (const T*)x_nchw, B, Cin, H, W,
                  (const T*)w_packed, (const T*)bias, Cout, (T*)out, (long long)ldo, extra...);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_conv_in(lb_ctx* ctx, const void* x_nchw, int B, int Cin, int H, int W, const void* w_packed,
                          const void* bias, int Cout, void* out, int64_t ldo, int act, float in_scale, void* stream,
                          int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_conv_in: unknown dtype %d", dtype);
    LB_REQUIRE(act == 0 || act == 1, "lb_conv_in: unknown act %d (0 = plain, 1 = tiny VAE input stage)", act);
    if (act == 1) {
        LB_REQUIRE(dtype == LB_DTYPE_F16, "lb_conv_in: the tiny VAE input stage (act 1) is fp16-only (dtype %d)", dtype);
        LB_REQUIRE(isfinite(in_scale), "lb_conv_in: in_scale must be finite");
        return conv_in_launch<__half, conv_in_tiny_kernel>(ctx, x_nchw, B, Cin, H, W, w_packed, bias, Cout, out, ldo,
                                                           stream, in_scale);
    }
    if (dtype == LB_DTYPE_BF16)
        return conv_in_launch<__nv_bfloat16, conv_in_kernel<__nv_bfloat16>>(ctx, x_nchw, B, Cin, H, W, w_packed, bias,
                                                                            Cout, out, ldo, stream);
    return conv_in_launch<__half, conv_in_kernel<__half>>(ctx, x_nchw, B, Cin, H, W, w_packed, bias, Cout, out, ldo,
                                                          stream);
}

extern "C" int lb_conv_in_add(lb_ctx* ctx, const void* x_nchw, int B, int Cin, int H, int W, const void* w_packed,
                              const void* bias, int Cout, void* out, int64_t ldo, const void* addend, int64_t ld_add,
                              void* stream) {
    LB_REQUIRE(addend && ld_add >= Cout && ld_add % 8 == 0 && lb_aligned16(addend),
               "lb_conv_in_add: addend needs a 16-byte aligned base and ld_add >= Cout, ld_add %% 8 == 0");
    return conv_in_launch<__half, conv_in_add_kernel>(ctx, x_nchw, B, Cin, H, W, w_packed, bias, Cout, out, ldo,
                                                      stream, (const __half*)addend, (long long)ld_add);
}

// the kernel moves 16-byte channel vectors, so fp16 and bf16 maps share it
extern "C" int lb_upsample_nearest(lb_ctx* ctx, const void* x, int64_t ld, int B, int H, int W, int C, void* out,
                                   int64_t ldo, int Ho, int Wo, void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_upsample_nearest: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && x && out, "lb_upsample_nearest: null argument");
    LB_REQUIRE(C % 8 == 0 && ld % 8 == 0 && ldo % 8 == 0, "lb_upsample_nearest: C and strides must be multiples of 8");
    LB_REQUIRE((Ho == 2 * H || Ho == 2 * H - 1) && (Wo == 2 * W || Wo == 2 * W - 1) && Ho >= 1 && Wo >= 1,
               "lb_upsample_nearest: output %dx%d is not a nearest 2x of %dx%d (need Ho in {2H-1, 2H}, Wo in {2W-1, 2W})",
               Ho, Wo, H, W);
    const long long total = (long long)B * Ho * Wo * (C / 8);
    lb_launch_pdl(upsample_nearest_kernel, grid_for(total, ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const __half*)x, ld, B, H, W, C, (__half*)out, ldo, Ho, Wo);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_im2col_s2(lb_ctx* ctx, const void* x, int64_t ld, int B, int H, int W, int C, void* out, void* stream) {
    LB_REQUIRE(ctx && x && out, "lb_im2col_s2: null argument");
    LB_REQUIRE(C % 8 == 0 && ld % 8 == 0, "lb_im2col_s2: C and stride must be multiples of 8");
    const long long total = (long long)B * ((H + 1) / 2) * ((W + 1) / 2) * 9 * (C / 8);
    lb_launch_pdl(im2col_s2_kernel<1>, grid_for(total, ctx->sm_count), kThreads, 0, lb_stream(stream), (const __half*)x, ld, B, H, W, C,
                                                                                        (__half*)out);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_im2col_s2_pad01(lb_ctx* ctx, const void* x, int64_t ld, int B, int H, int W, int C, void* out,
                                  void* stream) {
    LB_REQUIRE(ctx && x && out, "lb_im2col_s2_pad01: null argument");
    LB_REQUIRE(C % 8 == 0 && ld % 8 == 0 && ld >= C && lb_aligned16(x) && lb_aligned16(out),
               "lb_im2col_s2_pad01: C and stride must be multiples of 8, bases 16-byte aligned");
    LB_REQUIRE(B >= 1 && H >= 2 && W >= 2, "lb_im2col_s2_pad01: needs H, W >= 2 (got B %d H %d W %d)", B, H, W);
    const long long total = (long long)B * ((H - 2) / 2 + 1) * ((W - 2) / 2 + 1) * 9 * (C / 8);
    lb_launch_pdl(im2col_s2_kernel<0>, grid_for(total, ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const __half*)x, ld, B, H, W, C, (__half*)out);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_add_rows_bcast(lb_ctx* ctx, void* dst, int64_t ld_dst, const void* src, int64_t ld_src, int B,
                                 int64_t rows, int C, void* stream) {
    LB_REQUIRE(ctx && dst && src, "lb_add_rows_bcast: null argument");
    LB_REQUIRE(B >= 1 && rows >= 1 && C >= 8 && C % 8 == 0 && ld_dst % 8 == 0 && ld_src % 8 == 0 && ld_dst >= C &&
               ld_src >= C && lb_aligned16(dst) && lb_aligned16(src),
               "lb_add_rows_bcast: needs B, rows >= 1, C a multiple of 8, row strides >= C and multiples of 8, bases "
               "16-byte aligned (got B %d rows %lld C %d ld_dst %lld ld_src %lld)", B, (long long)rows, C,
               (long long)ld_dst, (long long)ld_src);
    const long long total = (long long)B * rows * (C / 8);
    lb_launch_pdl(add_rows_bcast_kernel, grid_for(total, ctx->sm_count), kThreads, 0, lb_stream(stream), (__half*)dst,
                  (long long)ld_dst, (const __half*)src, (long long)ld_src, B, (long long)rows, C);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_pixel_unshuffle_u8(lb_ctx* ctx, const void* img_u8, int H, int W, int Cimg, int r, void* out,
                                     void* stream) {
    LB_REQUIRE(ctx && img_u8 && out, "lb_pixel_unshuffle_u8: null argument");
    LB_REQUIRE(Cimg >= 1 && r >= 1 && (r * Cimg) % 8 == 0 && H >= r && W >= r && H % r == 0 && W % r == 0,
               "lb_pixel_unshuffle_u8: needs H, W multiples of r and r*Cimg a multiple of 8 (got H %d W %d Cimg %d "
               "r %d)", H, W, Cimg, r);
    LB_REQUIRE((reinterpret_cast<uintptr_t>(img_u8) & 7u) == 0 && lb_aligned16(out),
               "lb_pixel_unshuffle_u8: the image base must be 8-byte and the output base 16-byte aligned");
    const long long total = (long long)(H / r) * (W / r) * (r * r * Cimg / 8);
    lb_launch_pdl(pixel_unshuffle_u8_kernel, grid_for(total, ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const uint8_t*)img_u8, H, W, Cimg, r, (__half*)out);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_avgpool2_ceil(lb_ctx* ctx, const void* x, int64_t ld, int H, int W, int C, void* out, int64_t ldo,
                                void* stream) {
    LB_REQUIRE(ctx && x && out, "lb_avgpool2_ceil: null argument");
    LB_REQUIRE(H >= 1 && W >= 1 && C >= 8 && C % 8 == 0 && ld % 8 == 0 && ldo % 8 == 0 && ld >= C && ldo >= C &&
               lb_aligned16(x) && lb_aligned16(out),
               "lb_avgpool2_ceil: needs C a multiple of 8, row strides >= C and multiples of 8, bases 16-byte aligned "
               "(got H %d W %d C %d ld %lld ldo %lld)", H, W, C, (long long)ld, (long long)ldo);
    const long long total = (long long)((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
    lb_launch_pdl(avgpool2_ceil_kernel, grid_for(total, ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const __half*)x, (long long)ld, H, W, C, (__half*)out, (long long)ldo);
    LB_LAUNCH_CHECK();
    return 0;
}

// ======================= VAE-decoder helpers (SURVEY section 8f "next #1") ==========================================
// latent_prep: z = post_quant_conv(latents / scaling_factor), a per-pixel CxC matrix (diffusers_holder.py:135,
// AutoencoderKL.decode); NCHW fp16 in, fp16 or bf16 (TO) out, the 1/scaling_factor is folded into w on the host.
namespace {
template <typename TO>
__global__ void __launch_bounds__(kThreads)
latent_prep_kernel(const __half* __restrict__ x, int B, int C, long long hw, const float* __restrict__ w /*[C][C]*/,
                   const float* __restrict__ bias, TO* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)B * hw;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const long long b = i / hw, p = i % hw;
        float in[8];
        for (int c = 0; c < C; ++c) in[c] = __half2float(x[(b * C + c) * hw + p]);
        for (int o = 0; o < C; ++o) {
            float acc = bias[o];
            for (int c = 0; c < C; ++c) acc = fmaf(w[o * C + c], in[c], acc);
            out[(b * C + o) * hw + p] = LbType<TO>::from_f(acc);
        }
    }
}

// row softmax (in place capable): out[r,:] = softmax(x[r,:]) over `cols` fp16 values, one CTA per row.  Columns past
// the last multiple of 8 (h*w keys of a VAE latent with an odd side) take a scalar tail after the 128-bit loop.
// TO: the output type (fp16, or bf16 for the bf16 decoder's P); both are 2 bytes, so in place stays in place.
template <typename TO>
__global__ void __launch_bounds__(kThreads)
softmax_rows_kernel(const __half* __restrict__ x, long long ld, int cols, TO* __restrict__ out, long long ldo) {
    using L = LbType<TO>;
    pdl_launch_dependents();
    pdl_wait();
    const long long r = blockIdx.x;
    const __half* xr = x + r * ld;
    TO* orow = out + r * ldo;
    __shared__ float red[kThreads / 32];
    __shared__ float bc;
    const int vecs = cols >> 3;
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < vecs; v += kThreads) {
        const uint4 q = *reinterpret_cast<const uint4*>(xr + v * 8);
        const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h[j]);
            mx = fmaxf(mx, fmaxf(f.x, f.y));
        }
    }
    for (int c = (vecs << 3) + threadIdx.x; c < cols; c += kThreads) mx = fmaxf(mx, __half2float(xr[c]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = red[0];
        for (int i = 1; i < kThreads / 32; ++i) m = fmaxf(m, red[i]);
        bc = m;
    }
    __syncthreads();
    mx = bc;
    float sum = 0.f;
    for (int v = threadIdx.x; v < vecs; v += kThreads) {
        const uint4 q = *reinterpret_cast<const uint4*>(xr + v * 8);
        const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h[j]);
            sum += __expf(f.x - mx) + __expf(f.y - mx);
        }
    }
    for (int c = (vecs << 3) + threadIdx.x; c < cols; c += kThreads) sum += __expf(__half2float(xr[c]) - mx);
    sum = lb_warp_sum(sum);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < kThreads / 32; ++i) s += red[i];
        bc = 1.0f / s;
    }
    __syncthreads();
    const float inv = bc;
    for (int v = threadIdx.x; v < vecs; v += kThreads) {
        const uint4 q = *reinterpret_cast<const uint4*>(xr + v * 8);
        const __half2* h = reinterpret_cast<const __half2*>(&q);
        uint4 o;
        auto* oh = reinterpret_cast<typename L::T2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h[j]);
            oh[j] = L::from_f2(__expf(f.x - mx) * inv, __expf(f.y - mx) * inv);
        }
        *reinterpret_cast<uint4*>(orow + v * 8) = o;
    }
    for (int c = (vecs << 3) + threadIdx.x; c < cols; c += kThreads)
        orow[c] = L::from_f(__expf(__half2float(xr[c]) - mx) * inv);
}

// NHWC rows [B*hw, ld] (first C columns) -> NCHW [B, C, hw]: the boundary of the conv_out GEMM (C = 4 eps / 3 RGB
// channels out of an 8-column accumulator tile) back to the reference's tensor layout.
__global__ void __launch_bounds__(kThreads)
nhwc_to_nchw_kernel(const __half* __restrict__ x, long long ld, int B, int C, long long hw, __half* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)B * hw;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const long long b = i / hw, p = i % hw;
        const uint4 v = *reinterpret_cast<const uint4*>(x + i * ld);       // 8 channels of this pixel
        const __half* h = reinterpret_cast<const __half*>(&v);
        for (int c = 0; c < C; ++c) out[(b * C + c) * hw + p] = h[c];
    }
}

// VaeImageProcessor.postprocess: NCHW image -> uint8 NHWC, (x/2+0.5).clamp(0,1)*255 rounded half-to-even.
// Each instantiation follows the reference chain of its decoder.  fp16 (an fp16-safe VAE, or the tiny VAE): the
// reference decodes in fp16 and runs denormalize on that fp16 tensor, so x/2 and x/2 + 0.5 are each rounded to fp16
// before the clamp; * 255 and the rounding are fp32 (numpy).  bf16 (an upcast VAE): the reference decodes in fp32,
// so the whole chain is fp32.
// `nonfinite` (optional) counts NaN/Inf pixels: the decoder runs in fp16 where the reference upcasts the stock SDXL VAE
// to fp32 ("overflows in float16", diffusers_holder.py:128); an overflow anywhere upstream reaches the image as Inf/NaN.
template <typename T>
__global__ void __launch_bounds__(kThreads)
postprocess_u8_kernel(const T* __restrict__ img, int B, int C, long long hw, uint8_t* __restrict__ out,
                      int* __restrict__ nonfinite) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)B * hw * C;
    int bad = 0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const int c = (int)(i % C);
        const long long p = (i / C) % hw, b = i / (C * hw);
        const float raw = LbType<T>::to_f(img[(b * C + c) * hw + p]);
        bad += !isfinite(raw);
        float v;
        if constexpr (std::is_same<T, __half>::value) v = lb_round_h(lb_round_h(raw / 2.0f) + 0.5f);
        else v = raw / 2.0f + 0.5f;
        v = fminf(fmaxf(v, 0.f), 1.f);
        out[i] = (uint8_t)__float2int_rn(v * 255.0f);
    }
    if (nonfinite != nullptr && __any_sync(0xffffffffu, bad != 0)) {
        bad = __reduce_add_sync(0xffffffffu, bad);
        if ((threadIdx.x & 31) == 0) atomicAdd(nonfinite, bad);
    }
}
}  // namespace

extern "C" int lb_latent_prep(lb_ctx* ctx, const void* x_nchw, int B, int C, int64_t hw, const void* w_f32,
                              const void* bias_f32, void* out_nchw, void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_latent_prep: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && x_nchw && w_f32 && bias_f32 && out_nchw, "lb_latent_prep: null argument");
    LB_REQUIRE(C >= 1 && C <= 8, "lb_latent_prep: C must be <= 8");
    const unsigned grid = grid_for((long long)B * hw, ctx->sm_count);
    if (dtype == LB_DTYPE_BF16)
        lb_launch_pdl(latent_prep_kernel<__nv_bfloat16>, grid, kThreads, 0, lb_stream(stream), (const __half*)x_nchw, B,
                      C, hw, (const float*)w_f32, (const float*)bias_f32, (__nv_bfloat16*)out_nchw);
    else
        lb_launch_pdl(latent_prep_kernel<__half>, grid, kThreads, 0, lb_stream(stream), (const __half*)x_nchw, B, C, hw,
                      (const float*)w_f32, (const float*)bias_f32, (__half*)out_nchw);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_softmax_rows(lb_ctx* ctx, const void* x, int64_t ld, int64_t rows, int cols, void* out,
                               int64_t ldo, void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_softmax_rows: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && x && out, "lb_softmax_rows: null argument");
    LB_REQUIRE(cols >= 0 && ld % 8 == 0 && ldo % 8 == 0 && lb_aligned16(x) && lb_aligned16(out),
               "lb_softmax_rows: strides must be multiples of 8, bases 16B aligned");
    LB_REQUIRE(rows <= 2147483647LL, "lb_softmax_rows: too many rows");
    if (rows == 0) return 0;
    if (dtype == LB_DTYPE_BF16)
        lb_launch_pdl(softmax_rows_kernel<__nv_bfloat16>, (unsigned)rows, kThreads, 0, lb_stream(stream),
                      (const __half*)x, ld, cols, (__nv_bfloat16*)out, ldo);
    else
        lb_launch_pdl(softmax_rows_kernel<__half>, (unsigned)rows, kThreads, 0, lb_stream(stream), (const __half*)x, ld,
                      cols, (__half*)out, ldo);
    LB_LAUNCH_CHECK();
    return 0;
}

// copies 2-byte elements: the same kernel for fp16 and bf16
extern "C" int lb_nhwc_to_nchw(lb_ctx* ctx, const void* x, int64_t ld, int B, int C, int64_t hw, void* out_nchw,
                               void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_nhwc_to_nchw: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && x && out_nchw, "lb_nhwc_to_nchw: null argument");
    LB_REQUIRE(C >= 1 && C <= 8 && ld % 8 == 0 && ld >= 8 && lb_aligned16(x), "lb_nhwc_to_nchw: C <= 8, row stride a "
               "multiple of 8 elements, 16B aligned base");
    lb_launch_pdl(nhwc_to_nchw_kernel, grid_for((long long)B * hw, ctx->sm_count), kThreads, 0, lb_stream(stream),
                  (const __half*)x, (long long)ld, B, C, (long long)hw, (__half*)out_nchw);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_postprocess_u8(lb_ctx* ctx, const void* img_nchw, int B, int C, int64_t hw, void* out_u8_nhwc,
                                 int* nonfinite_count_dev, void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_postprocess_u8: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && img_nchw && out_u8_nhwc, "lb_postprocess_u8: null argument");
    const unsigned grid = grid_for((long long)B * hw * C, ctx->sm_count);
    if (dtype == LB_DTYPE_BF16)
        lb_launch_pdl(postprocess_u8_kernel<__nv_bfloat16>, grid, kThreads, 0, lb_stream(stream),
                      (const __nv_bfloat16*)img_nchw, B, C, hw, (uint8_t*)out_u8_nhwc, nonfinite_count_dev);
    else
        lb_launch_pdl(postprocess_u8_kernel<__half>, grid, kThreads, 0, lb_stream(stream), (const __half*)img_nchw, B, C,
                      hw, (uint8_t*)out_u8_nhwc, nonfinite_count_dev);
    LB_LAUNCH_CHECK();
    return 0;
}
