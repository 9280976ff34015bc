// gemm_sm90.cu -- K7/K4: wgmma GEMM and implicit-GEMM convolution for sm_90a.
//
//   out[M, N] = epilogue( sum_seg A_seg[M, K_seg] * W[N, K]^T )
//
// Replaces every dense contraction of the SDXL UNet the reference runs through
// cuBLAS / cuDNN (call site latentblending/diffusers_holder.py:336-344): the
// Linear layers (to_q/k/v, to_out, proj_in/out, GEGLU FF), the 3x3 / 1x1
// convolutions of the resnets and samplers (implicit GEMM: one K-segment per
// filter tap, the A tile of a tap is a TMA box of the NHWC activation shifted
// by (dy,dx) with hardware zero fill at the borders -- no im2col buffer), and
// the resnet shortcut folded in as an extra K-segment from a second tensor.
//
// Two M tilings (gemm_plan_build picks the one with fewer tiles; a tie keeps the box):
//   box  : a 128-row tile is a tw x th x tb box of pixels (128 x 1 x 1 when W >= 128; W and, if H*W < 128, H powers
//          of two otherwise), one tiled TMA load per k-block;
//   runs : tile m is rows [128 m, 128 m + 128) of the flattened pixel order, any W and H; one TMA im2col load per
//          k-block fetches the 128 pixels (across row and image boundaries) shifted by the filter tap.
// Both fill the same 128 x 128 B swizzled A tile, and every output element is the same k-ordered dot product, so
// the two give bit-identical results wherever both apply.
//
// Structure (one CTA per SM, persistent over 128 x BN output tiles, 384 threads = three warpgroups):
//   warpgroup 0   : TMA producer -- one warp issues cp.async.bulk.tensor 4D (A) / 2D (W) into a STAGES-deep
//                   128B-swizzled smem ring, mbarrier full/empty pairs, in the CTA's tile order; the warpgroup gives
//                   its registers away
//   warpgroups 1-2: consumers, ping-pong -- each owns whole 128-row tiles, alternating through the CTA's tiles
//                   (warpgroup 1: tiles 0, 2, 4, ...; warpgroup 2: tiles 1, 3, 5, ...).  Per k16 step two
//                   wgmma.m64nBNk16 (rows 0-63 and 64-127) share the B descriptor; fp16 in, fp32 accumulators in
//                   registers, one k-block in flight while the previous one's slot is released.  A pair of
//                   mbarriers lets one warpgroup at a time issue its main loop; the other meanwhile runs its epilogue
//                   straight from the accumulators: + bias / per-batch bias (time embedding) / residual, or GEGLU,
//                   or the LayerNorm fold, fp16 store.  So the tensor pipe keeps working through every epilogue
//                   but a CTA's last.
//                   BN = 256 (long-K convolutions only, see gemm_plan_build) does not fit one warpgroup's registers
//                   at 128 rows: there both warpgroups work on every tile, 64 rows each (cooperative).
// Weight (B operand) tiles of the first pipeline stages are requested BEFORE
// griddepcontrol.wait when the caller marks the weights static (LB_GEMM_STATIC_W):
// their HBM latency hides behind the tail of the previous kernel.
// Element type: fp16, or bf16 (LB_GEMM_BF16: the VAE decoder of a checkpoint whose activations overflow fp16) -- a
// template parameter that changes only the TMA element type, the wgmma input type and the epilogue's loads / stores
// (bf16 kernels: linear epilogue only; LB_GEMM_OUT_F16 stores fp16).  Both are 2 bytes, so boxes, swizzle, ring and
// tilings are shared.
// Depth-to-space (LB_GEMM_D2S2, gemm_tc_d2s_kernel): nearest-2x upsample + 3x3 conv as one GEMM over the
// low-resolution map -- N = 4 * Co phase filters, and the linear epilogue stores column p * Co + c of pixel (y, x) at
// upsampled pixel (2y + a, 2x + b), p = 2a + b (the tiny VAE decoder's upsampling convolutions).  The existing kernels
// instantiate the same body with the store off.
// Bound: tensor pipe; algorithmic FLOPs = 2*M*N*K.
#include "gemm_sm90.cuh"
#include <stdlib.h>

#include <type_traits>

#include "sm90.cuh"

using namespace sm90;

namespace {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kEpiParts = 4;                 // stats_out partial sums per row and N tile: one per lane of a quad
constexpr int kThreadsGemm = 384;            // warpgroup 0 TMA, warpgroups 1-2 wgmma + epilogue
constexpr int kABytes = kBM * kBK * 2;  // 16 KiB
constexpr int kGegluBN = 128;                // N tile of GEGLU launches (64 value + 64 gate columns)

template <int BN> struct Cfg {
    static constexpr int b_bytes = BN * kBK * 2;
    static constexpr int stage_bytes = kABytes + b_bytes;
    // ring depth: as many stages as 227 KB of shared memory allow
    static constexpr int stages = (BN <= 64) ? 8 : (BN <= 128) ? 7 : (BN <= 160) ? 6 : 4;
    // consumer schedule: ping-pong over whole tiles while a warpgroup's BN fp32 accumulators per thread fit its 232
    // registers (BN <= 160); cooperative (64 rows per warpgroup) for BN = 256
    static constexpr bool coop = BN > 160;
    static constexpr int smem_bytes = stages * stage_bytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(smem_bytes <= 227 * 1024, "smem ring does not fit");
};

// exact-erf GELU, 0.5 x (1 + erf(x / sqrt 2)), with erf from Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, far below
// the fp16 rounding the reference applies to gelu(gate)): ~14 FMA-pipe instructions + MUFU.RCP + MUFU.EX2 instead
// of erff's two-branch polynomial.
// For z < 0, 1 + erf(z) = erfc(|z|) is formed directly (no cancellation in the negative tail).
__device__ __forceinline__ float gelu_erf(float x) {
    const float z = fabsf(x) * 0.70710678118654752440f;
    const float t = __frcp_rn(fmaf(0.3275911f, z, 1.0f));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float erfc_abs = poly * t * exp2f(-1.4426950408889634f * z * z);     // erfc(|z|)
    const float one_plus_erf = x >= 0.f ? 2.0f - erfc_abs : erfc_abs;
    return 0.5f * x * one_plus_erf;
}

__device__ __forceinline__ float2 ld_f2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
template <typename T> __device__ __forceinline__ typename LbType<T>::T2 ld_2(const T* p) {
    return __ldg(reinterpret_cast<const typename LbType<T>::T2*>(p));
}

// (mu, rstd) of one row of the LayerNorm-folded A operand from the producer's per-row partial sums (fixed order).
// The partials of a row are contiguous (<= 64 x float2): they are fetched as float4 pairs, eight loads in flight at
// a time.
__device__ __forceinline__ void ln_row_stats(const GemmParams& p, long long row, bool ok, float& mu, float& rstd) {
    mu = 0.f;
    rstd = 1.f;
    if (!ok) return;
    float s = 0.f, q = 0.f;
    const float4* st = reinterpret_cast<const float4*>(p.ln_stats + row * p.ln_parts);   // ln_parts is even
    const int pairs = p.ln_parts >> 1;
    for (int base = 0; base < pairs; base += 8) {
        float4 v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = (base + i < pairs) ? __ldcg(st + base + i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            s += v[i].x;
            q += v[i].y;
            s += v[i].z;
            q += v[i].w;
        }
    }
    mu = s * p.ln_inv_k;
    double var = (double)q * (double)p.ln_inv_k - (double)mu * (double)mu;
    if (var < 0.0) var = 0.0;
    rstd = rsqrtf((float)var + p.ln_eps);
}

// One accumulator row of the current tile as the epilogue sees it.
struct EpiRow {
    long long row;     // output row (pixel index b*H*W + y*W + x)
    int bidx;          // batch index (bias2 row)
    bool ok;           // inside the output
    float ln_mu, ln_rstd;
};

// Epilogues of one 64-row half of the tile.  The thread holds rows r[0], r[1] (acc[4j + 2i + e] is row r[i], column
// 8j + 2*quad + e).  The global loads of a batch of column groups are all issued before any of its stores: the
// residual may alias the output (in-place `hs += f(hs)`) and only this thread reads and writes these elements, so
// the order is safe, and the loads overlap instead of costing one L2 round trip per 8-column group.
// T: the element type of bias, bias2, res and out (bf16 kernels store fp16 instead when p.out_f16 is set); the
// LayerNorm fold and stats_out exist in the fp16 kernels only.
// kD2S (LB_GEMM_D2S2, fp16 only): depth-to-space store.  Row r is low-resolution pixel (b, y, x) of a B x H x W map and
// column n = ph * Co + c (Co = p.d2s_co, ph = 2a + b') goes to output pixel (b, 2y + a, 2x + b'), channel c, of the
// B x 2H x 2W NHWC output.  Co % 8 == 0, so an 8-column group never straddles two phases; the phase of each group is
// tracked incrementally across the unrolled group loop (one division per row, none per group).
template <int BN, typename T, bool kD2S = false>
__device__ __forceinline__ void epilogue_linear(const GemmParams& p, const float (&acc)[BN / 2], const EpiRow (&r)[2],
                                                int n_tile, int quad) {
    using L = LbType<T>;
    using T2 = typename L::T2;
    constexpr bool kF16 = std::is_same<T, __half>::value;
    static_assert(!kD2S || kF16, "the depth-to-space epilogue is fp16-only");
    constexpr int G = BN / 8;                    // 8-column groups per row
    constexpr int CH = G > 10 ? G / 2 : G;       // groups per load batch (register budget)
    static_assert(G % CH == 0, "load batches must tile the row");
    const int n_base = n_tile * BN + 2 * quad;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (!r[i].ok) continue;
        float st_sum = 0.f, st_sq = 0.f;
        // (no residual, bias2, LayerNorm fold or stats_out with depth-to-space: rejected on the host)
        const T* res_row = (!kD2S && p.res) ? reinterpret_cast<const T*>(p.res) + r[i].row * p.ldr : nullptr;
        const T* b2_row =
            (!kD2S && p.bias2) ? reinterpret_cast<const T*>(p.bias2) + (long long)r[i].bidx * p.bias2_ld : nullptr;
        T* out_row = reinterpret_cast<T*>(p.out) + r[i].row * p.ldo;
        // depth-to-space: ph / cc are the phase and channel of the current group's first column (n_base - 2 quad);
        // d2s_px is the output row of phase 0 (b, 2y, 2x), d2s_row2 the row distance of phase a = 1 (one output row)
        int ph = 0, cc = 0;
        long long d2s_px = 0, d2s_row2 = 0;
        if constexpr (kD2S) {
            const int col0 = n_tile * BN;
            ph = col0 / p.d2s_co;
            cc = col0 - ph * p.d2s_co;
            const int W = p.W, HW = p.H * p.W;
            const int b = (int)(r[i].row / HW), rem = (int)(r[i].row - (long long)b * HW);
            const int y = rem / W, x = rem - y * W;
            d2s_row2 = 2LL * W;
            d2s_px = ((long long)b * 2 * p.H + 2 * y) * d2s_row2 + 2 * x;
        }
#pragma unroll
        for (int c0 = 0; c0 < G; c0 += CH) {
            float v[CH][2];
#pragma unroll
            for (int g = 0; g < CH; ++g) {
                v[g][0] = acc[4 * (c0 + g) + 2 * i];
                v[g][1] = acc[4 * (c0 + g) + 2 * i + 1];
            }
            if (!kD2S && kF16 && p.ln_stats) {
                constexpr int CL = CH > 8 ? CH / 2 : CH;     // fp32 vectors: half the batch
#pragma unroll
                for (int l0 = 0; l0 < CH; l0 += CL) {
                    float2 c[CL], t[CL];
#pragma unroll
                    for (int g = 0; g < CL; ++g) {
                        const int n = n_base + 8 * (c0 + l0 + g);
                        c[g] = n < p.N ? ld_f2(p.ln_csum + n) : make_float2(0.f, 0.f);
                        t[g] = n < p.N ? ld_f2(p.ln_bias + n) : make_float2(0.f, 0.f);
                    }
#pragma unroll
                    for (int g = 0; g < CL; ++g) {
                        v[l0 + g][0] = fmaf(r[i].ln_rstd, v[l0 + g][0] - r[i].ln_mu * c[g].x, t[g].x);
                        v[l0 + g][1] = fmaf(r[i].ln_rstd, v[l0 + g][1] - r[i].ln_mu * c[g].y, t[g].y);
                    }
                }
            } else {
                const T2 z = L::zero2();
                T2 hb[CH], hb2[CH], hr[CH];
#pragma unroll
                for (int g = 0; g < CH; ++g) {
                    const int n = n_base + 8 * (c0 + g);    // N is a multiple of 8 (checked on the host)
                    const bool in = n < p.N;
                    hb[g] = (p.bias && in) ? ld_2(reinterpret_cast<const T*>(p.bias) + n) : z;
                    hb2[g] = (b2_row && in) ? ld_2(b2_row + n) : z;
                    hr[g] = (res_row && in) ? *reinterpret_cast<const T2*>(res_row + n) : z;
                }
#pragma unroll
                for (int g = 0; g < CH; ++g) {
                    if (p.bias) {
                        const float2 t = L::to_f2(hb[g]);
                        v[g][0] += t.x;
                        v[g][1] += t.y;
                    }
                    if (b2_row) {
                        const float2 t = L::to_f2(hb2[g]);
                        v[g][0] += t.x;
                        v[g][1] += t.y;
                    }
                    if (res_row) {
                        const float2 t = L::to_f2(hr[g]);
                        v[g][0] += t.x;
                        v[g][1] += t.y;
                    }
                }
            }
#pragma unroll
            for (int g = 0; g < CH; ++g) {
                const int n = n_base + 8 * (c0 + g);
                if (n < p.N) {
                    float v0 = v[g][0], v1 = v[g][1];
                    if (p.relu) {
                        v0 = fmaxf(v0, 0.f);
                        v1 = fmaxf(v1, 0.f);
                    }
                    if constexpr (kD2S) {
                        const long long orow = d2s_px + (ph >> 1) * d2s_row2 + (ph & 1);
                        *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.out) + orow * p.ldo + cc + 2 * quad) =
                            __floats2half2_rn(v0, v1);
                    } else if constexpr (kF16) {
                        const __half2 o = __floats2half2_rn(v0, v1);
                        *reinterpret_cast<__half2*>(out_row + n) = o;
                        if (p.stats_out) {       // statistics of the STORED (fp16-rounded) values
                            const float2 f = __half22float2(o);
                            st_sum += f.x + f.y;
                            st_sq = fmaf(f.x, f.x, fmaf(f.y, f.y, st_sq));
                        }
                    } else if (p.out_f16) {      // the same 2-byte element address, fp16 value
                        *reinterpret_cast<__half2*>(out_row + n) = __floats2half2_rn(v0, v1);
                    } else {
                        *reinterpret_cast<T2*>(out_row + n) = L::from_f2(v0, v1);
                    }
                }
                if constexpr (kD2S) {
                    cc += 8;
                    if (cc == p.d2s_co) { cc = 0; ++ph; }
                }
            }
        }
        if (!kD2S && kF16 && p.stats_out)
            p.stats_out[r[i].row * (kEpiParts * p.tiles_n) + kEpiParts * n_tile + quad] = make_float2(st_sum, st_sq);
    }
}

// GEGLU: tile columns [0,BN/2) are "value", [BN/2,BN) the matching "gate" (weights are row-interleaved per tile on
// the host); out = (v+bv) * gelu(g+bg), BN/2 outputs per tile.
template <int BN>
__device__ __forceinline__ void epilogue_geglu(const GemmParams& p, const float (&acc)[BN / 2], const EpiRow (&r)[2],
                                               int n_tile, int quad) {
    constexpr int HN = BN / 2;
    constexpr int G = HN / 8;
    const int o_base = n_tile * HN + 2 * quad;     // output column base
    const int a_base = n_tile * BN + 2 * quad;     // accumulator (bias) column base
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (!r[i].ok) continue;
        __half* out_row = p.out + r[i].row * p.ldo;
        float2 bv[G], bg[G];
        if (p.ln_stats) {
            float2 cv[G], cg[G];
#pragma unroll
            for (int j = 0; j < G; ++j) {
                cv[j] = ld_f2(p.ln_csum + a_base + 8 * j);
                cg[j] = ld_f2(p.ln_csum + a_base + HN + 8 * j);
                bv[j] = ld_f2(p.ln_bias + a_base + 8 * j);
                bg[j] = ld_f2(p.ln_bias + a_base + HN + 8 * j);
            }
#pragma unroll
            for (int j = 0; j < G; ++j) {
                float v[2] = {acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]};
                float g[2] = {acc[4 * (j + G) + 2 * i], acc[4 * (j + G) + 2 * i + 1]};
                v[0] = r[i].ln_rstd * (v[0] - r[i].ln_mu * cv[j].x);
                v[1] = r[i].ln_rstd * (v[1] - r[i].ln_mu * cv[j].y);
                g[0] = r[i].ln_rstd * (g[0] - r[i].ln_mu * cg[j].x);
                g[1] = r[i].ln_rstd * (g[1] - r[i].ln_mu * cg[j].y);
                // the reference rounds proj output, gelu(gate) and the product to fp16
                const float r0 = lb_round_h(v[0] + bv[j].x) * lb_round_h(gelu_erf(lb_round_h(g[0] + bg[j].x)));
                const float r1 = lb_round_h(v[1] + bv[j].y) * lb_round_h(gelu_erf(lb_round_h(g[1] + bg[j].y)));
                *reinterpret_cast<__half2*>(out_row + o_base + 8 * j) = __floats2half2_rn(r0, r1);
            }
        } else {
#pragma unroll
            for (int j = 0; j < G; ++j) {
                bv[j] = p.bias ? __half22float2(ld_2(p.bias + a_base + 8 * j)) : make_float2(0.f, 0.f);
                bg[j] = p.bias ? __half22float2(ld_2(p.bias + a_base + HN + 8 * j)) : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int j = 0; j < G; ++j) {
                const float r0 = lb_round_h(acc[4 * j + 2 * i] + bv[j].x) *
                                 lb_round_h(gelu_erf(lb_round_h(acc[4 * (j + G) + 2 * i] + bg[j].x)));
                const float r1 = lb_round_h(acc[4 * j + 2 * i + 1] + bv[j].y) *
                                 lb_round_h(gelu_erf(lb_round_h(acc[4 * (j + G) + 2 * i + 1] + bg[j].y)));
                *reinterpret_cast<__half2*>(out_row + o_base + 8 * j) = __floats2half2_rn(r0, r1);
            }
        }
    }
}

// kRuns: pixel-run M tiles (p.runs = 1); a separate instantiation, so the pixel-box kernels stay as they were.
// T: operand / epilogue element type, __half or __nv_bfloat16 (LB_GEMM_BF16; linear epilogue only).
// kD2S: the depth-to-space store of LB_GEMM_D2S2 (its own kernels, gemm_tc_d2s_kernel, below).
template <int BN, bool kRuns, typename T, bool kD2S>
__device__ __forceinline__ void gemm_tc_body(const GemmParams& p) {
    using C = Cfg<BN>;
    constexpr bool kF16 = std::is_same<T, __half>::value;
    constexpr int nst = C::stages;
    constexpr bool kCoop = C::coop;
    pdl_launch_dependents();       // the next kernel may start its launch + prologue while this one runs
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);  // SWIZZLE_128B needs 1024 B alignment
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + nst * kABytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + nst * C::stage_bytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + nst;
    uint64_t* turn = bars + 2 * nst;   // ping-pong: turn[c] completes when consumer warpgroup c may issue its main loop

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const int wg = warp >> 2;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmA[0]);
        tma_prefetch_desc(&p.tmA[1]);
        tma_prefetch_desc(&p.tmB);
        for (int s = 0; s < nst; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], kCoop ? 2 : 1);       // released by every warpgroup that consumed the slot
        }
        mbar_init(&turn[0], 128);                        // every thread of the other warpgroup arrives
        mbar_init(&turn[1], 128);
        fence_mbar_init();
    }
    __syncthreads();

    const int m_groups = p.tiles_m;
    const int num_tiles = m_groups * p.tiles_n;
    const int tile0 = (int)blockIdx.x;
    const int tile_step = (int)gridDim.x;

    // Static weights do not depend on the previous grid: request the B tiles of the first ring stages now, while
    // that grid is still finishing (the A tiles of the same stages follow after griddepcontrol.wait).
    int early_kb = 0;
    if (p.static_w && tile0 < num_tiles) early_kb = p.total_kb < nst ? p.total_kb : nst;
    if (warp == 0 && early_kb > 0) {
        if (elect_one()) {
            const int n_tile = tile0 / m_groups;
            for (int kb = 0; kb < early_kb; ++kb) {
                mbar_expect_tx(&full[kb], C::stage_bytes);
                tma_load_2d(smem_b + kb * C::b_bytes, &p.tmB, &full[kb], kb * kBK, n_tile * BN);
            }
        }
        __syncwarp();
    }
    pdl_wait();                               // everything above overlapped the previous kernel; its outputs are visible now

    if (wg == 0) {
        reg_dealloc<40>();
        if (warp != 0) return;
        // ===================== TMA producer (whole warp runs the loop, one elected lane issues) =====================
        // The ring holds the CTA's tiles in order, which is the order the two consumer warpgroups take turns in.
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = tile0; tile < num_tiles; tile += tile_step) {
            const int m_tile = tile % m_groups, n_tile = tile / m_groups;
            // box: the tile's corner pixel (x0, y0, b0); runs: the pixel-box coordinate of the run's first pixel,
            // whose box starts one pixel up and left of the image (see encode_act_map_runs)
            int x0, y0, b0;
            if constexpr (kRuns) {
                const int row0 = m_tile * kBM;
                b0 = row0 / p.HW;
                const int rem = row0 - b0 * p.HW;
                y0 = rem / p.W - 1;
                x0 = rem % p.W - 1;
            } else {
                x0 = (m_tile % p.tiles_x) * p.tw;
                y0 = ((m_tile / p.tiles_x) % p.tiles_y) * p.th;
                b0 = (m_tile / (p.tiles_x * p.tiles_y)) * p.tb;
            }
            int kb_global = 0;
            for (int s = 0; s < p.num_segs; ++s) {
                const CUtensorMap* ma = &p.tmA[p.seg_map[s]];
                const int dy = p.seg_dy[s], dx = p.seg_dx[s];
                for (int kb = 0; kb < p.seg_kb[s]; ++kb, ++kb_global) {
                    mbar_wait(&empty[stage], phase ^ 1, p.err_flag, 1);
                    if (elect_one()) {
                        // filter tap (dy, dx) in {-1, 0, 1}^2: a box shifted by (dx, dy), or a run read at im2col
                        // offset (dx + 1, dy + 1)
                        const auto load_a = [&]() {
                            if constexpr (kRuns)
                                tma_load_4d_im2col(smem_a + stage * kABytes, ma, &full[stage], kb * kBK, x0, y0, b0,
                                                   (uint16_t)(dx + 1), (uint16_t)(dy + 1));
                            else
                                tma_load_4d(smem_a + stage * kABytes, ma, &full[stage], kb * kBK, x0 + dx, y0 + dy, b0);
                        };
                        if (tile == tile0 && kb_global < early_kb) {
                            // expect_tx and the weight tile were issued before griddepcontrol.wait
                            load_a();
                        } else {
                            mbar_expect_tx(&full[stage], C::stage_bytes);
                            load_a();
                            tma_load_2d(smem_b + stage * C::b_bytes, &p.tmB, &full[stage], kb_global * kBK, n_tile * BN);
                        }
                    }
                    __syncwarp();
                    if (++stage == nst) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== consumers
    // ping-pong (BN <= 160): warpgroup 1 takes the CTA's tiles 0, 2, 4, ..., warpgroup 2 tiles 1, 3, 5, ..., each
    //   computes all 128 rows of its tile;
    // cooperative (BN = 256, whose 128-row tile would not fit one warpgroup's registers): both take every tile,
    //   warpgroup 1 rows 0-63, warpgroup 2 rows 64-127.
    reg_alloc<232>();
    const int cw = wg - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int quad = lane & 3;
    const int my_tiles = tile0 < num_tiles ? (num_tiles - tile0 + tile_step - 1) / tile_step : 0;
    constexpr int kHalves = kCoop ? 1 : 2;   // 64-row halves of the tile this warpgroup computes
    float acc[kHalves][BN / 2];
    const auto half_of = [&](int hh) { return kCoop ? cw : hh; };
    for (int j = kCoop ? 0 : cw; j < my_tiles; j += kCoop ? 1 : 2) {
        const int tile = tile0 + j * tile_step;
        const int m_tile = tile % m_groups, n_tile = tile / m_groups;
        // this thread's accumulator rows inside the 128-row tile: 64h + 16*(warp%4) + lane/4 + 8i is er[hh][i]
        EpiRow er[kHalves][2];
        const auto row_of = [&](int hh, int i) {
            const int rr = half_of(hh) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
            EpiRow& e = er[hh][i];
            if constexpr (kRuns) {     // a run may span images: each row takes its own image's bias2 row
                const int row = m_tile * kBM + rr;
                e.ok = row < p.M;
                e.row = (unsigned)row;      // row >= 0: zero extension leaves no high word to keep live
                e.bidx = row / p.HW;
                return;
            }
            const int x = (m_tile % p.tiles_x) * p.tw + rr % p.tw;
            const int y = ((m_tile / p.tiles_x) % p.tiles_y) * p.th + (rr / p.tw) % p.th;
            const int b = (m_tile / (p.tiles_x * p.tiles_y)) * p.tb + rr / (p.tw * p.th);
            e.ok = (x < p.W) && (y < p.H) && (b < p.B);
            e.row = ((long long)b * p.H + y) * p.W + x;
            e.bidx = b;
        };
        // LayerNorm-fold row statistics: fetched before the main loop so their latency hides behind it
        float ln_mu[kHalves][2], ln_rstd[kHalves][2];
#pragma unroll
        for (int hh = 0; hh < kHalves; ++hh)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                ln_mu[hh][i] = 0.f;
                ln_rstd[hh][i] = 1.f;
                if (kF16 && p.ln_stats) {
                    row_of(hh, i);
                    ln_row_stats(p, er[hh][i].row, er[hh][i].ok, ln_mu[hh][i], ln_rstd[hh][i]);
                }
            }
        // this tile's k-blocks follow the j tiles before it in the ring
        const uint32_t it0 = (uint32_t)j * (uint32_t)p.total_kb;
        int stage = (int)(it0 % nst);
        uint32_t phase = (it0 / nst) & 1u;
        // The first wgmma ignores the accumulators' values; zeroing them anyway ends the previous tile's values at
        // its epilogue, so the epilogue may reuse their registers.
#pragma unroll
        for (int hh = 0; hh < kHalves; ++hh)
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[hh][i] = 0.f;
        // ---- main loop; in ping-pong, issued only once the other warpgroup has issued all of tile j - 1.  That
        // order also keeps every full[] barrier at most one phase behind the one this warpgroup waits for.
        // Tile j > 0 waits for completion (j - 1) / 2 of turn[cw] (the other warpgroup's tiles j - 1, j + 1, ...);
        // a bounded wait, so a protocol error traps instead of hanging the GPU.
        if (!kCoop && j > 0) {      // (the branch keeps the barrier address a compile-time offset)
            const uint32_t par = (uint32_t)((j - 1) >> 1) & 1u;
            if (cw == 0) mbar_wait(&turn[0], par, p.err_flag, 4);
            else mbar_wait(&turn[1], par, p.err_flag, 4);
        }
        int prev_stage = -1;
        for (int kb = 0; kb < p.total_kb; ++kb) {
            mbar_wait(&full[stage], phase, p.err_flag, 3);
            const uint32_t a_addr = smem_u32(smem_a + stage * kABytes);
            const uint32_t b_addr = smem_u32(smem_b + stage * C::b_bytes);
#pragma unroll
            for (int hh = 0; hh < kHalves; ++hh) fence_regs(acc[hh]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBK / 16; ++k) {
                const uint64_t bdesc = make_smem_desc_sw128(b_addr + k * 32, 16, 1024);
#pragma unroll
                for (int hh = 0; hh < kHalves; ++hh)
                    WgmmaSS<BN>::template mma<0, !kF16>(acc[hh],
                                                 make_smem_desc_sw128(a_addr + half_of(hh) * (64 * 128) + k * 32, 16,
                                                                      1024),
                                                 bdesc, (kb | k) != 0);
            }
            wgmma_commit();
            wgmma_wait<1>();
#pragma unroll
            for (int hh = 0; hh < kHalves; ++hh) fence_regs(acc[hh]);
            if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);
            prev_stage = stage;
            if (++stage == nst) { stage = 0; phase ^= 1; }
        }
        if (!kCoop && j + 1 < my_tiles) {     // the other warpgroup's turn
            if (cw == 0) mbar_arrive(&turn[1]);
            else mbar_arrive(&turn[0]);
        }
        wgmma_wait<0>();
#pragma unroll
        for (int hh = 0; hh < kHalves; ++hh) fence_regs(acc[hh]);
        if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);
        // Pixel runs form a half's rows just before its epilogue, which keeps them out of the other half's register
        // live range (the BN = 160 run kernel spills otherwise); the box kernels form all rows first.
        const auto rows_of_half = [&](int hh) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                row_of(hh, i);
                er[hh][i].ln_mu = ln_mu[hh][i];
                er[hh][i].ln_rstd = ln_rstd[hh][i];
            }
        };
        if constexpr (!kRuns) {
#pragma unroll
            for (int hh = 0; hh < kHalves; ++hh) rows_of_half(hh);
        }

        // ---- epilogue from registers (in ping-pong, overlapping the other warpgroup's main loop)
#pragma unroll
        for (int hh = 0; hh < kHalves; ++hh) {
            if constexpr (kRuns) rows_of_half(hh);
            if (p.mode == 0) epilogue_linear<BN, T, kD2S>(p, acc[hh], er[hh], n_tile, quad);
            else if constexpr (!kD2S && kF16 && BN == kGegluBN) epilogue_geglu<BN>(p, acc[hh], er[hh], n_tile, quad);
        }
    }
}

template <int BN, bool kRuns, typename T>
__global__ void __launch_bounds__(kThreadsGemm, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
    gemm_tc_body<BN, kRuns, T, false>(p);
}

// LB_GEMM_D2S2: nearest-2x upsample + 3x3 conv as one GEMM over the low-resolution map (fp16)
template <int BN, bool kRuns>
__global__ void __launch_bounds__(kThreadsGemm, 1) gemm_tc_d2s_kernel(const __grid_constant__ GemmParams p) {
    gemm_tc_body<BN, kRuns, __half, true>(p);
}

// ---- host side ------------------------------------------------------------------------

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int get_encode(lb_ctx* ctx, EncodeTiledFn* fn) {
    if (!ctx->tmap_encode) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qres;
        LB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres));
        LB_REQUIRE(f != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
        ctx->tmap_encode = f;
    }
    *fn = reinterpret_cast<EncodeTiledFn>(ctx->tmap_encode);
    return 0;
}

// TMA element type of the fp16 / bf16 kernels (both 2 bytes: boxes, strides and the swizzle are the same)
CUtensorMapDataType tma_dtype(bool bf16) {
    return bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

// 4-D NHWC activation map: dims (C, W, H, B), box (64, tw, th, tb), 128B swizzle, zero OOB fill.
int encode_act_map(lb_ctx* ctx, CUtensorMap* m, const void* base, int64_t ld, int C, int W, int H, int B, int tw,
                   int th, int tb, bool bf16) {
    EncodeTiledFn enc;
    if (int e = get_encode(ctx, &enc)) return e;
    LB_REQUIRE(lb_aligned16(base), "activation base must be 16-byte aligned");
    LB_REQUIRE(ld % 8 == 0 && ld >= C, "activation row stride must be a multiple of 8 elements and >= C");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * W, (cuuint64_t)ld * 2 * W * H};
    cuuint32_t box[4] = {(cuuint32_t)kBK, (cuuint32_t)tw, (cuuint32_t)th, (cuuint32_t)tb};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(m, tma_dtype(bf16), 4, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(activation C=%d W=%d H=%d B=%d ld=%lld box=%d,%d,%d) failed: %d",
               C, W, H, B, (long long)ld, tw, th, tb, (int)r);
    return 0;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

int get_encode_im2col(lb_ctx* ctx, EncodeIm2colFn* fn) {
    if (!ctx->tmap_encode_im2col) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qres;
        LB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f, cudaEnableDefault, &qres));
        LB_REQUIRE(f != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeIm2col not available");
        ctx->tmap_encode_im2col = f;
    }
    *fn = reinterpret_cast<EncodeIm2colFn>(ctx->tmap_encode_im2col);
    return 0;
}

// 4-D NHWC activation map for pixel-run tiles: dims (C, W, H, B), im2col mode, 128 pixels x 64 channels per load,
// 128B swizzle, zero OOB fill.  The pixel bounding box runs from (-1, -1) to (W - 2, H - 2) in (x, y): W x H positions
// per image, so a run of 128 consecutive box positions is 128 consecutive output pixels.  The position of output pixel
// (x, y) is (x - 1, y - 1); with im2col offset (dx + 1, dy + 1) it reads input pixel (x + dx, y + dy), the 3x3 tap
// (dy, dx) at padding 1 (a 1x1 segment uses offset (1, 1)).
int encode_act_map_runs(lb_ctx* ctx, CUtensorMap* m, const void* base, int64_t ld, int C, int W, int H, int B,
                        bool bf16) {
    EncodeIm2colFn enc;
    if (int e = get_encode_im2col(ctx, &enc)) return e;
    LB_REQUIRE(lb_aligned16(base), "activation base must be 16-byte aligned");
    LB_REQUIRE(ld % 8 == 0 && ld >= C, "activation row stride must be a multiple of 8 elements and >= C");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * W, (cuuint64_t)ld * 2 * W * H};
    const int lower[2] = {-1, -1}, upper[2] = {-1, -1};     // (W, H)
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(m, tma_dtype(bf16), 4, const_cast<void*>(base), dims, strides, lower, upper,
                     (cuuint32_t)kBK, (cuuint32_t)kBM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeIm2col(activation C=%d W=%d H=%d B=%d ld=%lld) failed: %d", C, W, H,
               B, (long long)ld, (int)r);
    return 0;
}

int encode_weight_map(lb_ctx* ctx, CUtensorMap* m, const void* base, int64_t ld, int64_t K, int N, int bn, bool bf16) {
    EncodeTiledFn enc;
    if (int e = get_encode(ctx, &enc)) return e;
    LB_REQUIRE(lb_aligned16(base), "weight base must be 16-byte aligned");
    LB_REQUIRE(ld % 8 == 0 && ld >= K, "weight row stride must be a multiple of 8 elements and >= K");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)bn};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, tma_dtype(bf16), 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weight K=%lld N=%d bn=%d) failed: %d", (long long)K, N, bn,
               (int)r);
    return 0;
}

bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// The pixel box of 128 rows for this shape; nullptr, or why the box cannot tile it.
const char* box_tiling(const GemmDesc& d, int* tw, int* th, int* tb) {
    if (d.W >= kBM || (d.H == 1 && d.B == 1)) {   // rows of a plain matrix: ragged tail is zero-filled by TMA
        *tw = kBM; *th = 1; *tb = 1;
        return nullptr;
    }
    if (!is_pow2(d.W)) return "W < 128 must be a power of two";
    *tw = d.W;
    *th = kBM / d.W;
    if (*th > d.H) {
        if (!is_pow2(d.H)) return "H must be a power of two when H*W < 128";
        *th = d.H;
    }
    *tb = kBM / (*tw * *th);
    return nullptr;
}

template <int BN, bool kRuns, typename T, bool kD2S> int launch_tiled(const GemmPlan& plan, cudaStream_t st) {
    void (*const kernel)(const GemmParams) = kD2S ? gemm_tc_d2s_kernel<BN, kRuns> : gemm_tc_kernel<BN, kRuns, T>;
    static bool attr_set = false;
    if (!attr_set) {
        LB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::smem_bytes));
        attr_set = true;
    }
    LB_CHECK_CUDA(lb_launch_pdl(kernel, dim3((unsigned)plan.grid), dim3(kThreadsGemm), (size_t)Cfg<BN>::smem_bytes, st,
                                plan.p));
    return 0;
}

template <int BN, typename T, bool kD2S = false> int launch_bn_t(const GemmPlan& plan, cudaStream_t st) {
    return plan.p.runs ? launch_tiled<BN, true, T, kD2S>(plan, st) : launch_tiled<BN, false, T, kD2S>(plan, st);
}

template <int BN> int launch_bn(const GemmPlan& plan, cudaStream_t st) {
    if (plan.d2s) return launch_bn_t<BN, __half, true>(plan, st);
    return plan.bf16 ? launch_bn_t<BN, __nv_bfloat16>(plan, st) : launch_bn_t<BN, __half>(plan, st);
}

}  // namespace

int gemm_plan_build(lb_ctx* ctx, const GemmDesc& d, GemmPlan* plan) {
    LB_REQUIRE(ctx && plan, "gemm: null ctx/plan");
    LB_REQUIRE(d.a0 && d.w && d.out, "gemm: null a0/w/out");
    LB_REQUIRE(d.B >= 1 && d.H >= 1 && d.W >= 1 && d.N >= 8, "gemm: bad shape B=%d H=%d W=%d N=%d", d.B, d.H, d.W, d.N);
    LB_REQUIRE(d.taps == 1 || d.taps == 9, "gemm: taps must be 1 or 9");
    LB_REQUIRE(d.a0_c % kBK == 0 && d.a0_c > 0, "gemm: a0 channels (%d) must be a multiple of 64", d.a0_c);
    LB_REQUIRE(d.a1 == nullptr || (d.a1_c % kBK == 0 && d.a1_c > 0), "gemm: a1 channels must be a multiple of 64");
    LB_REQUIRE(d.N % 8 == 0, "gemm: N (%d) must be a multiple of 8", d.N);
    LB_REQUIRE(d.out_ld % 8 == 0 && lb_aligned16(d.out), "gemm: out must be 16B aligned with ld %% 8 == 0");
    LB_REQUIRE(!d.res || (d.res_ld % 8 == 0 && lb_aligned16(d.res)), "gemm: residual alignment");
    LB_REQUIRE(!d.bias || lb_aligned16(d.bias), "gemm: bias alignment");
    LB_REQUIRE(!d.bias2 || (lb_aligned16(d.bias2) && d.bias2_ld % 8 == 0), "gemm: bias2 alignment");
    GemmParams& p = plan->p;
    memset(&p, 0, sizeof(p));
    LB_REQUIRE((d.mode & ~(0xff | LB_GEMM_STATIC_W | LB_GEMM_RELU | LB_GEMM_TILE_BOX | LB_GEMM_TILE_RUNS | LB_GEMM_BF16 |
                           LB_GEMM_OUT_F16 | LB_GEMM_D2S2)) == 0,
               "gemm: unknown mode flags 0x%x", d.mode);
    const bool bf16 = (d.mode & LB_GEMM_BF16) != 0;
    const bool d2s = (d.mode & LB_GEMM_D2S2) != 0;
    if (d2s) {
        LB_REQUIRE(d.taps == 9, "gemm: LB_GEMM_D2S2 needs a 3x3 convolution (taps = 9, got %d)", d.taps);
        LB_REQUIRE(d.N % 32 == 0, "gemm: LB_GEMM_D2S2 needs N %% 32 == 0 (4 phases x a multiple of 8 channels; got %d)",
                   d.N);
        LB_REQUIRE((d.mode & 0xff) == 0, "gemm: LB_GEMM_D2S2 supports the linear epilogue only (no GEGLU)");
        LB_REQUIRE(!bf16, "gemm: LB_GEMM_D2S2 is fp16-only (no LB_GEMM_BF16)");
        LB_REQUIRE(!d.res && !d.bias2 && !d.a1, "gemm: LB_GEMM_D2S2 takes no residual, bias2 or second input");
        LB_REQUIRE(!d.ln_stats && !d.stats_out, "gemm: LB_GEMM_D2S2 does not support the LayerNorm fold or stats_out");
    }
    plan->d2s = d2s;
    LB_REQUIRE(bf16 || !(d.mode & LB_GEMM_OUT_F16), "gemm: LB_GEMM_OUT_F16 needs LB_GEMM_BF16");
    if (bf16) {
        LB_REQUIRE((d.mode & 0xff) == 0, "gemm: LB_GEMM_BF16 supports the linear epilogue only (no GEGLU)");
        LB_REQUIRE(!d.ln_stats, "gemm: LB_GEMM_BF16 does not support the LayerNorm fold");
        LB_REQUIRE(!d.stats_out, "gemm: LB_GEMM_BF16 does not support stats_out");
    }
    plan->bf16 = bf16;
    const int force = d.mode & (LB_GEMM_TILE_BOX | LB_GEMM_TILE_RUNS);
    LB_REQUIRE(force != (LB_GEMM_TILE_BOX | LB_GEMM_TILE_RUNS), "gemm: LB_GEMM_TILE_BOX and LB_GEMM_TILE_RUNS exclude "
               "each other");
    // --- M tiling: the pixel box or pixel runs, whichever needs fewer 128-row tiles (a tie keeps the box)
    const int64_t M = (int64_t)d.B * d.H * d.W;
    const int64_t run_tiles = lb_ceil_div(M, kBM);
    int tw = kBM, th = 1, tb = 1;
    const char* box_err = box_tiling(d, &tw, &th, &tb);
    int64_t box_tiles = -1;
    if (!box_err) box_tiles = lb_ceil_div(d.W, tw) * lb_ceil_div(d.H, th) * lb_ceil_div(d.B, tb);
    bool runs;
    if (force == LB_GEMM_TILE_BOX) {
        LB_REQUIRE(!box_err, "gemm: the pixel box cannot tile B=%d H=%d W=%d: %s", d.B, d.H, d.W, box_err);
        runs = false;
    } else if (force == LB_GEMM_TILE_RUNS) {
        runs = true;
    } else {
        runs = box_err != nullptr || run_tiles < box_tiles;
    }
    p.W = d.W; p.H = d.H; p.B = d.B;
    p.runs = runs ? 1 : 0;
    if (runs) {
        LB_REQUIRE(M <= 0x7fffffff, "gemm: pixel runs need B*H*W < 2^31 (got %lld)", (long long)M);
        p.M = (int)M;
        p.HW = d.H * d.W;
        p.tw = kBM; p.th = 1; p.tb = 1;
        p.tiles_x = p.tiles_y = 1;
        p.tiles_m = (int)run_tiles;
    } else {
        p.tw = tw; p.th = th; p.tb = tb;
        p.tiles_x = (int)lb_ceil_div(d.W, tw);
        p.tiles_y = (int)lb_ceil_div(d.H, th);
        p.tiles_m = (int)box_tiles;
    }
    // --- N tiling
    int bn;
    if ((d.mode & 0xff) == 1) {
        bn = kGegluBN;      // the weight rows are interleaved per 128-row N tile by the caller
        LB_REQUIRE(d.N % bn == 0, "gemm: GEGLU needs N %% %d == 0 (got %d)", bn, d.N);
    } else if (d.N % 256 == 0 && d.N >= 512 && (int64_t)(d.taps * d.a0_c + (d.a1 ? d.a1_c : 0)) >= 4096 &&
               (int64_t)p.tiles_m * (d.N / 256) >= 2 * ctx->sm_count) {
        // Long-K, many-tile convolutions (VAE decoder at 512 channels, the 64^2 upsample conv at batch 4): the
        // epilogue is a small share of a tile, and N = 256 wgmmas read less shared memory per FLOP than the
        // ping-pong tiles, so the cooperative 128 x 256 tile is faster there (measured per shape on H100).
        bn = 256;
    } else if (d.N % 160 == 0) bn = 160;
    else if (d.N % 128 == 0) bn = 128;
    else if (d.N <= 64) bn = 64;
    else bn = 128;
    plan->bn = bn;
    p.tiles_n = (int)lb_ceil_div(d.N, bn);
    p.N = d.N;
    LB_REQUIRE((d.mode & 0xff) <= 1, "gemm: unknown epilogue mode %d", d.mode & 0xff);
    p.mode = d.mode & 0xff;
    p.static_w = (d.mode & LB_GEMM_STATIC_W) ? 1 : 0;
    // --- K segments
    int ns = 0, total = 0;
    if (d.taps == 9) {
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx) {
                p.seg_map[ns] = 0; p.seg_dy[ns] = ky - 1; p.seg_dx[ns] = kx - 1; p.seg_kb[ns] = d.a0_c / kBK;
                total += p.seg_kb[ns++];
            }
    } else {
        p.seg_map[ns] = 0; p.seg_dy[ns] = 0; p.seg_dx[ns] = 0; p.seg_kb[ns] = d.a0_c / kBK;
        total += p.seg_kb[ns++];
    }
    if (d.a1) {
        p.seg_map[ns] = 1; p.seg_dy[ns] = 0; p.seg_dx[ns] = 0; p.seg_kb[ns] = d.a1_c / kBK;
        total += p.seg_kb[ns++];
    }
    p.num_segs = ns;
    p.total_kb = total;
    const int64_t Ktot = (int64_t)total * kBK;
    const auto encode_a = [&](CUtensorMap* m, const void* base, int64_t ld, int c) {
        return runs ? encode_act_map_runs(ctx, m, base, ld, c, d.W, d.H, d.B, bf16)
                    : encode_act_map(ctx, m, base, ld, c, d.W, d.H, d.B, tw, th, tb, bf16);
    };
    if (int e = encode_a(&p.tmA[0], d.a0, d.a0_ld, d.a0_c)) return e;
    if (d.a1) {
        if (int e = encode_a(&p.tmA[1], d.a1, d.a1_ld, d.a1_c)) return e;
    } else {
        p.tmA[1] = p.tmA[0];
    }
    if (int e = encode_weight_map(ctx, &p.tmB, d.w, d.w_ld, Ktot, d.N, bn, bf16)) return e;
    p.out = static_cast<__half*>(d.out);
    p.ldo = d.out_ld;
    p.out_f16 = (d.mode & LB_GEMM_OUT_F16) ? 1 : 0;
    p.d2s_co = d2s ? d.N / 4 : 0;
    p.bias = static_cast<const __half*>(d.bias);
    p.bias2 = static_cast<const __half*>(d.bias2);
    p.bias2_ld = d.bias2_ld;
    p.res = static_cast<const __half*>(d.res);
    p.ldr = d.res_ld;
    p.err_flag = lb_err_flag(ctx);
    p.relu = (d.mode & LB_GEMM_RELU) ? 1 : 0;
    LB_REQUIRE(!p.relu || p.mode == 0, "gemm: LB_GEMM_RELU needs the linear epilogue");
    if (d.ln_stats) {
        LB_REQUIRE(d.ln_csum && d.ln_bias && d.ln_parts >= 1 && d.ln_parts <= 64, "gemm: LayerNorm fold needs ln_csum, "
                   "ln_bias and 1 <= ln_parts <= 64");
        LB_REQUIRE(d.taps == 1 && !d.a1 && !d.res && !d.bias2 && !d.bias, "gemm: LayerNorm fold applies to a plain linear "
                   "(its bias is part of ln_bias)");
        LB_REQUIRE(lb_aligned16(d.ln_csum) && lb_aligned16(d.ln_bias) && lb_aligned16(d.ln_stats), "gemm: ln_* alignment");
        p.ln_stats = static_cast<const float2*>(d.ln_stats);
        p.ln_parts = d.ln_parts;
        p.ln_csum = static_cast<const float*>(d.ln_csum);
        p.ln_bias = static_cast<const float*>(d.ln_bias);
        p.ln_inv_k = 1.0f / (float)d.a0_c;
        p.ln_eps = d.ln_eps;
    }
    if (d.stats_out) {
        LB_REQUIRE(p.mode == 0, "gemm: stats_out needs the linear epilogue");
        LB_REQUIRE(d.stats_parts == kEpiParts * p.tiles_n, "gemm: stats_parts must be %d * ceil(N / %d) = %d (got %d)",
                   kEpiParts, bn, kEpiParts * p.tiles_n, d.stats_parts);
        p.stats_out = static_cast<float2*>(d.stats_out);
    }
    {
        const int tiles = p.tiles_m * p.tiles_n;
        plan->grid = tiles < ctx->sm_count ? tiles : ctx->sm_count;
    }
    return 0;
}

int gemm_plan_launch(const GemmPlan& plan, cudaStream_t st) {
    switch (plan.bn) {
        case 64: return launch_bn<64>(plan, st);
        case 128: return launch_bn<128>(plan, st);
        case 160: return launch_bn<160>(plan, st);
        case 256: return launch_bn<256>(plan, st);
    }
    lb_set_error("gemm: unsupported N tile %d", plan.bn);
    return 2;
}

extern "C" int lb_gemm_stats_parts(lb_ctx* ctx, const lb_gemm_desc* desc) {
    if (!ctx || !desc) return -1;
    GemmDesc d = *reinterpret_cast<const GemmDesc*>(desc);
    d.stats_out = nullptr;
    GemmPlan plan;
    if (gemm_plan_build(ctx, d, &plan)) return -1;
    return kEpiParts * plan.p.tiles_n;
}

extern "C" int lb_gemm(lb_ctx* ctx, const lb_gemm_desc* desc, void* stream) {
    LB_REQUIRE(ctx && desc, "lb_gemm: null argument");
    static_assert(sizeof(GemmDesc) == sizeof(lb_gemm_desc), "GemmDesc / lb_gemm_desc layout drift");
    GemmPlan plan;
    if (int e = gemm_plan_build(ctx, *reinterpret_cast<const GemmDesc*>(desc), &plan)) return e;
    return gemm_plan_launch(plan, lb_stream(stream));
}
