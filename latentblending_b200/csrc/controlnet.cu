// controlnet.cu -- the conditioning-image embedding of an SDXL ControlNet (diffusers 0.25
// ControlNetConditioningEmbedding): 3x3 pad-1 convolutions with few channels (3 -> 16 -> 32 -> 96 -> 256) at the
// full image resolution, stride 1 or 2, bias and SiLU fused, NHWC fp16 out.  The first layer reads the uint8 RGB
// control image and fuses the pipeline's ``/ 255`` (VaeImageProcessor without normalisation).
//
// These shapes do not fit lb_gemm (K = 9*Cin is not a multiple of 64, and an im2col of the 1024^2 layers would take
// ~400 MB), and the embedding runs once per control image, so a direct convolution is enough: one thread per output
// pixel and 8 output channels, the block's [9*Cin][8] weight slice in shared memory.
//
// The same kernel is the first convolution of the VAE encoder (diffusers 0.25 Encoder.conv_in, 3 -> 128): it reads
// the uint8 RGB image with VaeImageProcessor.preprocess fused (fp32 u / 255, then 2x - 1, one rounding to the
// encoder's storage type) and writes fp16 or bf16.  That layer runs once per image, and its K = 27 suits lb_gemm no
// better than the embedding's.
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kMaxCin = 256;

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

// how the kernel reads its input x
enum CondIn {
    kInF16 = 0,      // NHWC fp16 rows
    kInU8 = 1,       // uint8 image, u -> h(u / 255): the control image
    kInImage = 2     // uint8 image, u -> round_TO(2 (u / 255) - 1): VaeImageProcessor.preprocess before the VAE encoder
};

// TO: the element type of the weights, the bias and the output (fp16; fp16 or bf16 for kInImage)
template <int kIn, typename TO>
__global__ void __launch_bounds__(kThreads)
cond_conv_kernel(const void* __restrict__ x_raw, long long ld_x, int B, int H, int W, int Cin,
                 const TO* __restrict__ wp, const TO* __restrict__ bias, int Cout, int stride, int silu,
                 TO* __restrict__ out, long long ldo, int Ho, int Wo) {
    using L = LbType<TO>;
    using T2 = typename L::T2;
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ __half s_raw[];
    TO* s_w = reinterpret_cast<TO*>(s_raw);      // [9*Cin][8]: this block's 8 output channels
    const int g = blockIdx.y;
    const int rows = 9 * Cin;
    for (int i = threadIdx.x; i < rows; i += kThreads)
        *reinterpret_cast<uint4*>(s_w + i * 8) = *reinterpret_cast<const uint4*>(wp + (long long)i * Cout + g * 8);
    __syncthreads();
    const long long npix = (long long)B * Ho * Wo;
    const long long pix = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (pix >= npix) return;
    const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int ky = 0; ky < 3; ++ky) {
        const int yy = yo * stride + ky - 1;
        if (yy < 0 || yy >= H) continue;
        for (int kx = 0; kx < 3; ++kx) {
            const int xx = xo * stride + kx - 1;
            if (xx < 0 || xx >= W) continue;
            const long long ipix = ((long long)b * H + yy) * W + xx;
            const TO* wt = s_w + (ky * 3 + kx) * Cin * 8;
            if constexpr (kIn != kInF16) {
                const uint8_t* xp = reinterpret_cast<const uint8_t*>(x_raw) + ipix * ld_x;
                for (int c = 0; c < Cin; ++c) {
                    float xv;
                    if constexpr (kIn == kInU8) {
                        xv = lb_round_h((float)xp[c] / 255.0f);
                    } else {
                        const float u = (float)xp[c] / 255.0f;
                        xv = L::round(__fadd_rn(2.0f * u, -1.0f));     // 2u is exact: no fused multiply-add
                    }
                    const uint4 wv = *reinterpret_cast<const uint4*>(wt + c * 8);
                    const T2* wh = reinterpret_cast<const T2*>(&wv);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float2 f = L::to_f2(wh[j]);
                        acc[2 * j] = fmaf(xv, f.x, acc[2 * j]);
                        acc[2 * j + 1] = fmaf(xv, f.y, acc[2 * j + 1]);
                    }
                }
            } else {
                const __half* xp = reinterpret_cast<const __half*>(x_raw) + ipix * ld_x;
                for (int c0 = 0; c0 < Cin; c0 += 8) {
                    const uint4 xv8 = *reinterpret_cast<const uint4*>(xp + c0);
                    const __half* xh = reinterpret_cast<const __half*>(&xv8);
#pragma unroll
                    for (int cc = 0; cc < 8; ++cc) {
                        const float xv = __half2float(xh[cc]);
                        const uint4 wv = *reinterpret_cast<const uint4*>(wt + (c0 + cc) * 8);
                        const T2* wh = reinterpret_cast<const T2*>(&wv);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float2 f = L::to_f2(wh[j]);
                            acc[2 * j] = fmaf(xv, f.x, acc[2 * j]);
                            acc[2 * j + 1] = fmaf(xv, f.y, acc[2 * j + 1]);
                        }
                    }
                }
            }
        }
    }
    const uint4 bv = *reinterpret_cast<const uint4*>(bias + g * 8);
    const T2* bh = reinterpret_cast<const T2*>(&bv);
    float y[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 f = L::to_f2(bh[j]);
        y[2 * j] = L::round(acc[2 * j] + f.x);
        y[2 * j + 1] = L::round(acc[2 * j + 1] + f.y);
    }
    if (silu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = L::round(silu_f(y[j]));
    }
    uint4 o;
    T2* oh = reinterpret_cast<T2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) oh[j] = L::from_f2(y[2 * j], y[2 * j + 1]);
    *reinterpret_cast<uint4*>(out + pix * ldo + g * 8) = o;
}

}  // namespace

extern "C" int lb_cond_conv(lb_ctx* ctx, const void* x, int64_t ld_x, int B, int H, int W, int Cin, int in_u8,
                            const void* w_packed, const void* bias, int Cout, int stride, int silu, void* out,
                            int64_t ldo, void* stream) {
    LB_REQUIRE(ctx && x && w_packed && bias && out, "lb_cond_conv: null argument");
    LB_REQUIRE(B >= 1 && H >= 1 && W >= 1, "lb_cond_conv: bad sizes B %d H %d W %d", B, H, W);
    LB_REQUIRE(stride == 1 || stride == 2, "lb_cond_conv: stride must be 1 or 2 (got %d)", stride);
    LB_REQUIRE(silu == 0 || silu == 1, "lb_cond_conv: silu must be 0 or 1 (got %d)", silu);
    LB_REQUIRE(in_u8 == 0 || in_u8 == 1, "lb_cond_conv: in_u8 must be 0 or 1 (got %d)", in_u8);
    if (in_u8) {
        LB_REQUIRE(Cin >= 1 && Cin <= 8 && ld_x >= Cin, "lb_cond_conv: a uint8 input has 1 to 8 channels and ld_x >= Cin");
    } else {
        LB_REQUIRE(Cin >= 8 && Cin <= kMaxCin && Cin % 8 == 0 && ld_x >= Cin && ld_x % 8 == 0 && lb_aligned16(x),
                   "lb_cond_conv: an fp16 input needs Cin %% 8 == 0, 8 <= Cin <= %d, ld_x %% 8 == 0 and a 16-byte "
                   "aligned base (Cin %d, ld_x %lld)", kMaxCin, Cin, (long long)ld_x);
    }
    LB_REQUIRE(Cout >= 8 && Cout % 8 == 0 && ldo >= Cout && ldo % 8 == 0 && lb_aligned16(out) &&
                   lb_aligned16(w_packed) && lb_aligned16(bias),
               "lb_cond_conv: Cout %% 8 == 0, ldo %% 8 == 0 and 16-byte aligned w / bias / out required (Cout %d)", Cout);
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;      // floor((H + 2 - 3) / stride) + 1
    const long long npix = (long long)B * Ho * Wo;
    LB_REQUIRE(npix < (1LL << 31) * kThreads, "lb_cond_conv: too many output pixels");
    const dim3 grid((unsigned)lb_ceil_div(npix, kThreads), (unsigned)(Cout / 8));
    const size_t smem = (size_t)9 * Cin * 8 * sizeof(__half);
    cudaStream_t st = lb_stream(stream);
    if (in_u8)
        lb_launch_pdl(cond_conv_kernel<kInU8, __half>, grid, kThreads, smem, st, x, (long long)ld_x, B, H, W, Cin,
                      (const __half*)w_packed, (const __half*)bias, Cout, stride, silu, (__half*)out, (long long)ldo,
                      Ho, Wo);
    else
        lb_launch_pdl(cond_conv_kernel<kInF16, __half>, grid, kThreads, smem, st, x, (long long)ld_x, B, H, W, Cin,
                      (const __half*)w_packed, (const __half*)bias, Cout, stride, silu, (__half*)out, (long long)ldo,
                      Ho, Wo);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_image_conv_in(lb_ctx* ctx, const void* img_u8, int64_t ld_x, int B, int H, int W, int Cin,
                                const void* w_packed, const void* bias, int Cout, void* out, int64_t ldo, void* stream,
                                int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_image_conv_in: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && img_u8 && w_packed && bias && out, "lb_image_conv_in: null argument");
    LB_REQUIRE(B >= 1 && H >= 1 && W >= 1, "lb_image_conv_in: bad sizes B %d H %d W %d", B, H, W);
    LB_REQUIRE(Cin >= 1 && Cin <= 8 && ld_x >= Cin, "lb_image_conv_in: the image has 1 to 8 channels and ld_x >= Cin "
               "(Cin %d, ld_x %lld)", Cin, (long long)ld_x);
    LB_REQUIRE(Cout >= 8 && Cout % 8 == 0 && ldo >= Cout && ldo % 8 == 0 && lb_aligned16(out) &&
                   lb_aligned16(w_packed) && lb_aligned16(bias),
               "lb_image_conv_in: Cout %% 8 == 0, ldo %% 8 == 0 and 16-byte aligned w / bias / out required (Cout %d)",
               Cout);
    const long long npix = (long long)B * H * W;
    LB_REQUIRE(npix < (1LL << 31) * kThreads, "lb_image_conv_in: too many output pixels");
    const dim3 grid((unsigned)lb_ceil_div(npix, kThreads), (unsigned)(Cout / 8));
    const size_t smem = (size_t)9 * Cin * 8 * 2;
    cudaStream_t st = lb_stream(stream);
    if (dtype == LB_DTYPE_BF16)
        lb_launch_pdl(cond_conv_kernel<kInImage, __nv_bfloat16>, grid, kThreads, smem, st, img_u8, (long long)ld_x, B,
                      H, W, Cin, (const __nv_bfloat16*)w_packed, (const __nv_bfloat16*)bias, Cout, 1, 0,
                      (__nv_bfloat16*)out, (long long)ldo, H, W);
    else
        lb_launch_pdl(cond_conv_kernel<kInImage, __half>, grid, kThreads, smem, st, img_u8, (long long)ld_x, B, H, W,
                      Cin, (const __half*)w_packed, (const __half*)bias, Cout, 1, 0, (__half*)out, (long long)ldo, H,
                      W);
    LB_LAUNCH_CHECK();
    return 0;
}
