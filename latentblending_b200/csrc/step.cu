// step.cu -- K9: the scheduler arithmetic around the UNet call, fused.
//
// Replaces (per denoise step) latentblending/diffusers_holder.py:328-330
// (CFG duplicate + scheduler.scale_model_input), :347-349 (CFG combine),
// :356 (scheduler.step -- diffusers 0.25.0 Euler / Euler-ancestral) and :359
// (trajectory clone): ~14 torch elementwise kernels -> 2 launches.
//
// Parity contract: the reference stack rounds to fp16 after EVERY torch op
// (fp32 op-math with the fp32 0-dim sigma, fp16 store).  The fused kernels keep
// values in registers but apply the same roundings, so results are bit-identical
// to the op-by-op oracle (oracle/schedulers.py, oracle/holder.py).
// HBM-bound: (2B+1) reads + 2 writes of n fp16 elements.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float h(float x) { return lb_round_h(x); }

__global__ void __launch_bounds__(kThreads)
scale_input_kernel(const __half* __restrict__ x, __half* __restrict__ out, int64_t n, int batch, float divisor) {
    pdl_launch_dependents();
    pdl_wait();
    if (n % 8 == 0) {                      // 128-bit path (host checked the alignment)
        const int64_t nv = n / 8;
        for (int64_t v = (int64_t)blockIdx.x * kThreads + threadIdx.x; v < nv; v += (int64_t)gridDim.x * kThreads) {
            const uint4 vx = reinterpret_cast<const uint4*>(x)[v];
            const __half* hx = reinterpret_cast<const __half*>(&vx);
            uint4 vo;
            __half* ho = reinterpret_cast<__half*>(&vo);
#pragma unroll
            for (int e = 0; e < 8; ++e) ho[e] = __float2half_rn(__fdiv_rn(__half2float(hx[e]), divisor));
            for (int b = 0; b < batch; ++b) reinterpret_cast<uint4*>(out + (int64_t)b * n)[v] = vo;
        }
        return;
    }
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        __half v = __float2half_rn(__fdiv_rn(__half2float(x[i]), divisor));
        for (int b = 0; b < batch; ++b) out[(int64_t)b * n + i] = v;
    }
}

__device__ __forceinline__ float step_elem(float x, float eu, float et, float nz, bool use_cfg, bool has_noise,
                                           float g, float sigma, float dt, float sigma_up) {
    float e = eu;
    if (use_cfg) {
        float d = h(__fsub_rn(et, eu));   // noise_pred_text - noise_pred_uncond
        float m = h(__fmul_rn(g, d));     // guidance_scale * (...)
        e = h(__fadd_rn(eu, m));          // noise_pred_uncond + ...
    }
    float a = h(__fmul_rn(sigma, e));     // sigma * model_output
    float pred = h(__fsub_rn(x, a));      // pred_original_sample
    float d1 = h(__fsub_rn(x, pred));     // sample - pred_original_sample
    float deriv = h(__fdiv_rn(d1, sigma));
    float ee = h(__fmul_rn(deriv, dt));
    float xn = h(__fadd_rn(x, ee));
    if (has_noise) {
        float nn = h(__fmul_rn(nz, sigma_up));
        xn = h(__fadd_rn(xn, nn));
    }
    return xn;
}

__global__ void __launch_bounds__(kThreads)
cfg_euler_kernel(const __half* __restrict__ x, const __half* __restrict__ eps, const __half* __restrict__ eps_text,
                 const __half* __restrict__ noise,
                 __half* __restrict__ out, __half* __restrict__ traj, int64_t n, int use_cfg, float g,
                 float sigma, float dt, float sigma_up, __half* __restrict__ scaled_next, int scaled_batch,
                 float next_divisor) {
    pdl_launch_dependents();
    pdl_wait();
    const bool has_noise = noise != nullptr;
    const bool vec = (n % 8 == 0);
    if (vec) {
        const int64_t nv = n / 8;
        for (int64_t v = (int64_t)blockIdx.x * kThreads + threadIdx.x; v < nv; v += (int64_t)gridDim.x * kThreads) {
            uint4 vx = reinterpret_cast<const uint4*>(x)[v];
            uint4 vu = lb_ldg_stream(reinterpret_cast<const uint4*>(eps) + v);
            uint4 vt = use_cfg ? lb_ldg_stream(reinterpret_cast<const uint4*>(eps_text) + v) : vu;
            uint4 vn = has_noise ? lb_ldg_stream(reinterpret_cast<const uint4*>(noise) + v) : make_uint4(0, 0, 0, 0);
            const __half* hx = reinterpret_cast<const __half*>(&vx);
            const __half* hu = reinterpret_cast<const __half*>(&vu);
            const __half* ht = reinterpret_cast<const __half*>(&vt);
            const __half* hn = reinterpret_cast<const __half*>(&vn);
            uint4 vo;
            __half* ho = reinterpret_cast<__half*>(&vo);
#pragma unroll
            for (int e = 0; e < 8; ++e)
                ho[e] = __float2half_rn(step_elem(__half2float(hx[e]), __half2float(hu[e]), __half2float(ht[e]),
                                                  __half2float(hn[e]), use_cfg != 0, has_noise, g, sigma, dt,
                                                  sigma_up));
            reinterpret_cast<uint4*>(out)[v] = vo;
            if (traj) reinterpret_cast<uint4*>(traj)[v] = vo;
            if (scaled_next) {               // next step's scale_model_input + CFG duplicate, same roundings as the op
                uint4 vs;
                __half* hs = reinterpret_cast<__half*>(&vs);
#pragma unroll
                for (int e = 0; e < 8; ++e) hs[e] = __float2half_rn(__fdiv_rn(__half2float(ho[e]), next_divisor));
                for (int b = 0; b < scaled_batch; ++b) reinterpret_cast<uint4*>(scaled_next + (int64_t)b * n)[v] = vs;
            }
        }
    } else {
        for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
            float r = step_elem(__half2float(x[i]), __half2float(eps[i]),
                                use_cfg ? __half2float(eps_text[i]) : 0.f, has_noise ? __half2float(noise[i]) : 0.f,
                                use_cfg != 0, has_noise, g, sigma, dt, sigma_up);
            out[i] = __float2half_rn(r);
            if (traj) traj[i] = __float2half_rn(r);
            if (scaled_next) {
                const __half sv = __float2half_rn(__fdiv_rn(__half2float(__float2half_rn(r)), next_divisor));
                for (int b = 0; b < scaled_batch; ++b) scaled_next[(int64_t)b * n + i] = sv;
            }
        }
    }
}

}  // namespace

extern "C" int lb_scale_model_input(lb_ctx* ctx, const void* latents, void* out, int64_t n, int batch,
                                    float divisor, void* stream) {
    LB_REQUIRE(ctx != nullptr, "lb_scale_model_input: null context");
    LB_REQUIRE(latents && out, "lb_scale_model_input: null buffer");
    LB_REQUIRE(batch >= 1 && n > 0, "lb_scale_model_input: bad sizes");
    if (n % 8 == 0) LB_REQUIRE(lb_aligned16(latents) && lb_aligned16(out), "lb_scale_model_input: 16-byte alignment");
    unsigned grid = (unsigned)lb_ceil_div(n, n % 8 == 0 ? (int64_t)kThreads * 8 : (int64_t)kThreads);
    if (grid > (unsigned)ctx->sm_count * 8) grid = (unsigned)ctx->sm_count * 8;
    lb_launch_pdl(scale_input_kernel, grid, kThreads, 0, lb_stream(stream), (const __half*)latents, (__half*)out, n, batch,
                                                                divisor);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_cfg_euler_step(lb_ctx* ctx, const void* latents, const void* eps, const void* eps_text,
                                 const void* noise, void* out,
                                 void* traj, int64_t n, int use_cfg, float guidance, float sigma, float dt,
                                 float sigma_up, void* scaled_next, int scaled_batch, float next_divisor,
                                 void* stream) {
    LB_REQUIRE(ctx != nullptr, "lb_cfg_euler_step: null context");
    LB_REQUIRE(latents && eps && out, "lb_cfg_euler_step: null buffer");
    LB_REQUIRE(n > 0, "lb_cfg_euler_step: n must be positive");
    LB_REQUIRE(!scaled_next || (scaled_batch >= 1 && next_divisor > 0.f), "lb_cfg_euler_step: scaled_next needs a batch "
               "and a positive divisor");
    if (n % 8 == 0)
        LB_REQUIRE(lb_aligned16(latents) && lb_aligned16(eps) && lb_aligned16(out) &&
                       (!noise || lb_aligned16(noise)) && (!traj || lb_aligned16(traj)) &&
                       (!scaled_next || lb_aligned16(scaled_next)),
                   "lb_cfg_euler_step: buffers must be 16-byte aligned");
    unsigned grid = (unsigned)lb_ceil_div(n, (int64_t)kThreads * 8);
    if (grid > (unsigned)ctx->sm_count * 8) grid = (unsigned)ctx->sm_count * 8;
    if (grid < 1) grid = 1;
    const __half* et = eps_text ? (const __half*)eps_text : (const __half*)eps + n;   // default: [2,n] = (uncond, text)
    LB_REQUIRE(n % 8 != 0 || lb_aligned16(et), "lb_cfg_euler_step: eps_text must be 16-byte aligned");
    lb_launch_pdl(cfg_euler_kernel, grid, kThreads, 0, lb_stream(stream), (const __half*)latents, (const __half*)eps, et,
                                                              (const __half*)noise, (__half*)out, (__half*)traj, n,
                                                              use_cfg, guidance, sigma, dt, sigma_up,
                                                              (__half*)scaled_next, scaled_batch, next_divisor);
    LB_LAUNCH_CHECK();
    return 0;
}
