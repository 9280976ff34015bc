// step.cu -- K9: the scheduler arithmetic around the UNet call, fused.
//
// Replaces (per denoise step) latentblending/diffusers_holder.py:328-330
// (CFG duplicate + scheduler.scale_model_input), :347-349 (CFG combine),
// :356 (scheduler.step -- diffusers 0.25.0 Euler / Euler-ancestral / LCM / DPM-Solver++ multistep) and :359
// (trajectory clone): ~14 torch elementwise kernels -> 2 launches.  One kernel template
// (cfg_step_kernel) carries the I/O; the scheduler's per-element update is its parameter.  A multistep update
// (DPM-Solver++) also reads the previous step's x0 prediction and writes this step's, one buffer per branch.
//
// Parity contract: the reference stack rounds to fp16 after EVERY torch op
// (fp32 op-math with the fp32 0-dim sigma, fp16 store).  The fused kernels keep
// values in registers but apply the same roundings, so results are bit-identical
// to the op-by-op oracle (oracle/schedulers.py, oracle/holder.py).
// HBM-bound: (2B+1) reads + 2 writes of n fp16 elements.
//
// add_noise_rows_kernel starts a trajectory part-way down the schedule from an image's latents (img2img): every
// forward-diffused row the denoise loop skips, plus its start latent, in one launch (scheduler.add_noise of diffusers
// 0.25.0 on fp16 CUDA tensors, with the same fp16 roundings).
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

// The per-element scheduler updates.  Each takes the CFG-combined eps and returns the new latent (fp32 holding an
// fp16 value); the skeleton below (loads, CFG combine, stores, fused next-step input) is shared by all of them.  An
// update with kHistory also takes the previous step's x0 (when has_prev) and returns this step's through ``x0``.
constexpr int kStepScalars = 7;

struct EulerUpdate {          // diffusers 0.25.0 EulerDiscreteScheduler / EulerAncestralDiscreteScheduler.step
    static constexpr bool kHistory = false;
    float sigma, dt, sigma_up;
    __device__ __forceinline__ static EulerUpdate make(const float (&s)[kStepScalars]) {
        return EulerUpdate{s[0], s[1], s[2]};
    }
    __device__ __forceinline__ float operator()(float x, float e, float nz, bool has_noise) const {
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
};

struct LcmUpdate {            // diffusers 0.25.0 LCMScheduler.step, epsilon prediction
    static constexpr bool kHistory = false;
    float sb, inv_sa, c_skip, c_out, sap, sbp;
    __device__ __forceinline__ static LcmUpdate make(const float (&s)[kStepScalars]) {
        return LcmUpdate{s[0], s[1], s[2], s[3], s[4], s[5]};
    }
    __device__ __forceinline__ float operator()(float x, float e, float nz, bool has_noise) const {
        float a = h(__fmul_rn(sb, e));        // beta_prod_t.sqrt() * model_output
        float d = h(__fsub_rn(x, a));         // sample - ...
        float x0 = h(__fmul_rn(d, inv_sa));   // ... / alpha_prod_t.sqrt(): a CPU scalar divisor is a reciprocal multiply
        float p = h(__fmul_rn(c_out, x0));    // c_out * predicted_original_sample
        float q = h(__fmul_rn(c_skip, x));    // c_skip * sample
        float den = h(__fadd_rn(p, q));       // denoised
        if (has_noise) {                      // every step but the last
            float u = h(__fmul_rn(sap, den)); // alpha_prod_t_prev.sqrt() * denoised
            float v = h(__fmul_rn(sbp, nz));  // beta_prod_t_prev.sqrt() * noise
            den = h(__fadd_rn(u, v));
        }
        return den;
    }
};

// diffusers 0.25.0 DPMSolverMultistepScheduler.step, dpmsolver++ / sde-dpmsolver++, epsilon prediction, first order
// or the multistep second order (midpoint / heun).  The host folds the solver variant and the signs of the
// subtracted terms into c_x, c_0, c_1, c_n (negating a product before rounding is exact).
struct DpmUpdate {
    static constexpr bool kHistory = true;
    float sigma_s, inv_alpha_s, inv_r0, c_x, c_0, c_1, c_n;
    __device__ __forceinline__ static DpmUpdate make(const float (&s)[kStepScalars]) {
        return DpmUpdate{s[0], s[1], s[2], s[3], s[4], s[5], s[6]};
    }
    __device__ __forceinline__ float operator()(float x, float e, float nz, bool has_noise, float x0p, bool has_prev,
                                                float& x0) const {
        float a = h(__fmul_rn(sigma_s, e));    // sigma_t * model_output        (convert_model_output)
        float d = h(__fsub_rn(x, a));          // sample - ...
        x0 = h(__fmul_rn(d, inv_alpha_s));     // ... / alpha_t: a CPU scalar divisor is a reciprocal multiply
        float xn = h(__fadd_rn(h(__fmul_rn(c_x, x)), h(__fmul_rn(c_0, x0))));
        if (has_prev) {                        // second order; a never-written history may hold NaN, so skip it
            float d1 = h(__fmul_rn(inv_r0, h(__fsub_rn(x0, x0p))));   // (1 / r0) * (m0 - m1)
            xn = h(__fadd_rn(xn, h(__fmul_rn(c_1, d1))));
        }
        if (has_noise) xn = h(__fadd_rn(xn, h(__fmul_rn(c_n, nz))));  // sde-dpmsolver++
        return xn;
    }
};

template <class Update>
__device__ __forceinline__ float step_elem(const Update& upd, float x, float eu, float et, float nz, bool use_cfg,
                                           bool has_noise, float g, float x0p, bool has_prev, float& x0) {
    float e = eu;
    if (use_cfg) {
        float d = h(__fsub_rn(et, eu));   // noise_pred_text - noise_pred_uncond
        float m = h(__fmul_rn(g, d));     // guidance_scale * (...)
        e = h(__fadd_rn(eu, m));          // noise_pred_uncond + ...
    }
    if constexpr (Update::kHistory) return upd(x, e, nz, has_noise, x0p, has_prev, x0);
    else return upd(x, e, nz, has_noise);
}

// The update's scalars s0..s6 are separate float parameters (an Update that needs fewer leaves the rest unread); the
// first three keep the offsets the Euler kernel has always had.  x0_prev / x0_out (kHistory updates only; NULL
// x0_prev: first order) are not __restrict__: x0_out may alias x0_prev, each element read before the same thread
// writes it.
template <class Update>
__global__ void __launch_bounds__(kThreads)
cfg_step_kernel(const __half* __restrict__ x, const __half* __restrict__ eps, const __half* __restrict__ eps_text,
                const __half* __restrict__ noise,
                __half* __restrict__ out, __half* __restrict__ traj, int64_t n, int use_cfg, float g,
                float s0, float s1, float s2, __half* __restrict__ scaled_next, int scaled_batch, float next_divisor,
                float s3, float s4, float s5, float s6, const __half* x0_prev, __half* x0_out) {
    pdl_launch_dependents();
    pdl_wait();
    const Update upd = Update::make({s0, s1, s2, s3, s4, s5, s6});
    const bool has_noise = noise != nullptr;
    const bool has_prev = Update::kHistory && x0_prev != nullptr;
    const bool vec = (n % 8 == 0);
    if (vec) {
        const int64_t nv = n / 8;
        for (int64_t v = (int64_t)blockIdx.x * kThreads + threadIdx.x; v < nv; v += (int64_t)gridDim.x * kThreads) {
            uint4 vx = reinterpret_cast<const uint4*>(x)[v];
            uint4 vu = lb_ldg_stream(reinterpret_cast<const uint4*>(eps) + v);
            uint4 vt = use_cfg ? lb_ldg_stream(reinterpret_cast<const uint4*>(eps_text) + v) : vu;
            uint4 vn = has_noise ? lb_ldg_stream(reinterpret_cast<const uint4*>(noise) + v) : make_uint4(0, 0, 0, 0);
            uint4 vp = has_prev ? reinterpret_cast<const uint4*>(x0_prev)[v] : make_uint4(0, 0, 0, 0);
            const __half* hx = reinterpret_cast<const __half*>(&vx);
            const __half* hu = reinterpret_cast<const __half*>(&vu);
            const __half* ht = reinterpret_cast<const __half*>(&vt);
            const __half* hn = reinterpret_cast<const __half*>(&vn);
            const __half* hp = reinterpret_cast<const __half*>(&vp);
            uint4 vo, v0;
            __half* ho = reinterpret_cast<__half*>(&vo);
            __half* h0 = reinterpret_cast<__half*>(&v0);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                float x0 = 0.f;
                ho[e] = __float2half_rn(step_elem(upd, __half2float(hx[e]), __half2float(hu[e]), __half2float(ht[e]),
                                                  __half2float(hn[e]), use_cfg != 0, has_noise, g,
                                                  __half2float(hp[e]), has_prev, x0));
                h0[e] = __float2half_rn(x0);
            }
            reinterpret_cast<uint4*>(out)[v] = vo;
            if (traj) reinterpret_cast<uint4*>(traj)[v] = vo;
            if (Update::kHistory) reinterpret_cast<uint4*>(x0_out)[v] = v0;
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
            float x0 = 0.f;
            float r = step_elem(upd, __half2float(x[i]), __half2float(eps[i]),
                                use_cfg ? __half2float(eps_text[i]) : 0.f, has_noise ? __half2float(noise[i]) : 0.f,
                                use_cfg != 0, has_noise, g, has_prev ? __half2float(x0_prev[i]) : 0.f, has_prev, x0);
            if (Update::kHistory) x0_out[i] = __float2half_rn(x0);
            out[i] = __float2half_rn(r);
            if (traj) traj[i] = __float2half_rn(r);
            if (scaled_next) {
                const __half sv = __float2half_rn(__fdiv_rn(__half2float(__float2half_rn(r)), next_divisor));
                for (int b = 0; b < scaled_batch; ++b) scaled_next[(int64_t)b * n + i] = sv;
            }
        }
    }
}

// Host side shared by the step entry points: argument checks, the default eps_text (the text half right after the
// unconditional one in a [2,n] eps) and the launch.
template <class Update>
int launch_cfg_step(const char* name, lb_ctx* ctx, const void* latents, const void* eps, const void* eps_text,
                    const void* noise, void* out, void* traj, int64_t n, int use_cfg, float guidance,
                    const float (&s)[kStepScalars], void* scaled_next, int scaled_batch, float next_divisor,
                    void* stream, const void* x0_prev = nullptr, void* x0_out = nullptr) {
    LB_REQUIRE(ctx != nullptr, "%s: null context", name);
    LB_REQUIRE(latents && eps && out, "%s: null buffer", name);
    LB_REQUIRE(n > 0, "%s: n must be positive", name);
    LB_REQUIRE(!scaled_next || (scaled_batch >= 1 && next_divisor > 0.f), "%s: scaled_next needs a batch "
               "and a positive divisor", name);
    if (n % 8 == 0)
        LB_REQUIRE(lb_aligned16(latents) && lb_aligned16(eps) && lb_aligned16(out) &&
                       (!noise || lb_aligned16(noise)) && (!traj || lb_aligned16(traj)) &&
                       (!scaled_next || lb_aligned16(scaled_next)) && (!x0_prev || lb_aligned16(x0_prev)) &&
                       (!x0_out || lb_aligned16(x0_out)),
                   "%s: buffers must be 16-byte aligned", name);
    unsigned grid = (unsigned)lb_ceil_div(n, (int64_t)kThreads * 8);
    if (grid > (unsigned)ctx->sm_count * 8) grid = (unsigned)ctx->sm_count * 8;
    if (grid < 1) grid = 1;
    const __half* et = eps_text ? (const __half*)eps_text : (const __half*)eps + n;   // default: [2,n] = (uncond, text)
    LB_REQUIRE(n % 8 != 0 || lb_aligned16(et), "%s: eps_text must be 16-byte aligned", name);
    lb_launch_pdl(cfg_step_kernel<Update>, grid, kThreads, 0, lb_stream(stream), (const __half*)latents,
                  (const __half*)eps, et, (const __half*)noise, (__half*)out, (__half*)traj, n, use_cfg, guidance, s[0], s[1],
                  s[2], (__half*)scaled_next, scaled_batch, next_divisor, s[3], s[4], s[5], s[6],
                  (const __half*)x0_prev, (__half*)x0_out);
    LB_LAUNCH_CHECK();
    return 0;
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
    const float s[kStepScalars] = {sigma, dt, sigma_up, 0.f, 0.f, 0.f, 0.f};
    return launch_cfg_step<EulerUpdate>("lb_cfg_euler_step", ctx, latents, eps, eps_text, noise, out, traj, n, use_cfg,
                                        guidance, s, scaled_next, scaled_batch, next_divisor, stream);
}

extern "C" int lb_cfg_lcm_step(lb_ctx* ctx, const void* latents, const void* eps, const void* eps_text,
                               const void* noise, void* out, void* traj, int64_t n, int use_cfg, float guidance,
                               float sqrt_beta, float inv_sqrt_alpha, float c_skip, float c_out,
                               float sqrt_alpha_prev, float sqrt_beta_prev, void* scaled_next, int scaled_batch,
                               float next_divisor, void* stream) {
    const float s[kStepScalars] = {sqrt_beta, inv_sqrt_alpha, c_skip, c_out, sqrt_alpha_prev, sqrt_beta_prev, 0.f};
    return launch_cfg_step<LcmUpdate>("lb_cfg_lcm_step", ctx, latents, eps, eps_text, noise, out, traj, n, use_cfg,
                                      guidance, s, scaled_next, scaled_batch, next_divisor, stream);
}

extern "C" int lb_cfg_dpm_step(lb_ctx* ctx, const void* latents, const void* eps, const void* eps_text,
                               const void* noise, const void* x0_prev, void* x0_out, void* out, void* traj, int64_t n,
                               int use_cfg, float guidance, float sigma_s, float inv_alpha_s, float inv_r0, float c_x,
                               float c_0, float c_1, float c_n, void* scaled_next, int scaled_batch,
                               float next_divisor, void* stream) {
    LB_REQUIRE(x0_out != nullptr, "lb_cfg_dpm_step: x0_out (this step's x0, the branch's history) is required");
    const float s[kStepScalars] = {sigma_s, inv_alpha_s, inv_r0, c_x, c_0, c_1, c_n};
    return launch_cfg_step<DpmUpdate>("lb_cfg_dpm_step", ctx, latents, eps, eps_text, noise, out, traj, n, use_cfg,
                                      guidance, s, scaled_next, scaled_batch, next_divisor, stream, x0_prev, x0_out);
}

namespace {

// out[r] = add_noise(x0, eps, coeffs[r]), every op rounded to fp16 like the reference's fp16 tensors (h = rounding):
//   form 0 (Euler, Euler-ancestral):  h(x + h(eps * b))             x0 + noise * sigma
//   form 1 (LCM, DPM-Solver++):       h(h(a * x) + h(b * eps))      sqrt_alpha * x0 + sqrt_one_minus_alpha * noise
// x = h(x0): a bf16 x0 is rounded to fp16 first (the pipeline's .to(fp16)).  Each thread reads x0 and eps once and
// writes every row.  `nonfinite` (optional) counts the non-finite x0 elements.
template <typename TX>
__global__ void __launch_bounds__(kThreads)
add_noise_rows_kernel(const TX* __restrict__ x0, const __half* __restrict__ eps, const __half* __restrict__ coeffs,
                      int form, long long n, int rows, __half* __restrict__ out, int* __restrict__ nonfinite) {
    pdl_launch_dependents();
    pdl_wait();
    int bad = 0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const float xr = LbType<TX>::to_f(x0[i]);
        bad += !isfinite(xr);
        const float x = h(xr);
        const float e = __half2float(eps[i]);
        for (int r = 0; r < rows; ++r) {
            const float a = __half2float(coeffs[2 * r]), b = __half2float(coeffs[2 * r + 1]);
            const float v = form == 0 ? h(x + h(e * b)) : h(h(a * x) + h(b * e));
            out[(long long)r * n + i] = __float2half_rn(v);
        }
    }
    if (nonfinite != nullptr && __any_sync(0xffffffffu, bad != 0)) {
        bad = __reduce_add_sync(0xffffffffu, bad);
        if ((threadIdx.x & 31) == 0) atomicAdd(nonfinite, bad);
    }
}

}  // namespace

extern "C" int lb_add_noise_rows(lb_ctx* ctx, const void* x0, const void* noise, const void* coeffs_dev, int form,
                                 int64_t n, int rows, void* out, int* nonfinite_count_dev, void* stream, int dtype) {
    LB_REQUIRE(dtype == LB_DTYPE_F16 || dtype == LB_DTYPE_BF16, "lb_add_noise_rows: unknown dtype %d", dtype);
    LB_REQUIRE(ctx && x0 && noise, "lb_add_noise_rows: null argument");
    LB_REQUIRE(form == 0 || form == 1, "lb_add_noise_rows: unknown form %d (0 = x0 + b*noise, 1 = a*x0 + b*noise)", form);
    LB_REQUIRE(n > 0 && rows >= 0, "lb_add_noise_rows: bad sizes n %lld rows %d", (long long)n, rows);
    LB_REQUIRE(rows == 0 || (coeffs_dev && out), "lb_add_noise_rows: rows > 0 needs coeffs and out");
    unsigned grid = (unsigned)lb_ceil_div(n, (int64_t)kThreads);
    if (grid > (unsigned)ctx->sm_count * 8) grid = (unsigned)ctx->sm_count * 8;
    if (dtype == LB_DTYPE_BF16)
        lb_launch_pdl(add_noise_rows_kernel<__nv_bfloat16>, grid, kThreads, 0, lb_stream(stream),
                      (const __nv_bfloat16*)x0, (const __half*)noise, (const __half*)coeffs_dev, form, (long long)n,
                      rows, (__half*)out, nonfinite_count_dev);
    else
        lb_launch_pdl(add_noise_rows_kernel<__half>, grid, kThreads, 0, lb_stream(stream), (const __half*)x0,
                      (const __half*)noise, (const __half*)coeffs_dev, form, (long long)n, rows, (__half*)out,
                      nonfinite_count_dev);
    LB_LAUNCH_CHECK();
    return 0;
}
