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
// Structure (one CTA per SM, persistent over 128 x BN output tiles, 384 threads = three warpgroups):
//   warpgroup 0   : TMA producer -- one warp issues cp.async.bulk.tensor 4D (A) / 2D (W) into a STAGES-deep
//                   128B-swizzled smem ring, mbarrier full/empty pairs; the warpgroup gives its registers away
//   warpgroups 1-2: consumers    -- each owns 64 rows of the tile: wgmma.m64nBNk16 (fp16 in, fp32 accumulators in
//                   registers, one k-block in flight while the previous one's slot is released), then the
//                   epilogue straight from the accumulators: + bias / per-batch bias (time embedding) / residual,
//                   or GEGLU, or the LayerNorm fold, fp16 store.  The producer runs ahead into the next tile's
//                   k-blocks while the consumers drain the epilogue.
// Weight (B operand) tiles of the first pipeline stages are requested BEFORE
// griddepcontrol.wait when the caller marks the weights static (LB_GEMM_STATIC_W):
// their HBM latency hides behind the tail of the previous kernel.
// Bound: tensor pipe; algorithmic FLOPs = 2*M*N*K.
#include "gemm_sm90.cuh"
#include <stdlib.h>

#include "sm90.cuh"

using namespace sm90;

namespace {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kEpiParts = 4;                 // stats_out partial sums per row and N tile: one per lane of a quad
constexpr int kThreadsGemm = 384;            // warpgroup 0 TMA, warpgroups 1-2 wgmma + epilogue
constexpr int kABytes = kBM * kBK * 2;  // 16 KiB

template <int BN> struct Cfg {
    static constexpr int b_bytes = BN * kBK * 2;
    static constexpr int stage_bytes = kABytes + b_bytes;
    // ring depth (GemmParams::stages): as many stages as 227 KB of shared memory allow
    static constexpr int deep = (BN <= 64) ? 8 : (BN <= 128) ? 7 : (BN <= 160) ? 6 : 4;
    static constexpr int smem_bytes(int nst) { return nst * stage_bytes + 1024 /*align slack*/ + 256 /*barriers*/; }
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

__device__ __forceinline__ float2 ld_h2(const __half* p) {
    return __half22float2(__ldg(reinterpret_cast<const __half2*>(p)));
}
__device__ __forceinline__ float2 ld_f2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

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

template <int BN>
__global__ void __launch_bounds__(kThreadsGemm, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
    using C = Cfg<BN>;
    pdl_launch_dependents();       // the next kernel may start its launch + prologue while this one runs
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);  // SWIZZLE_128B needs 1024 B alignment
    uint8_t* smem_a = smem;
    const int nst = p.stages;      // ring depth (Cfg::deep)
    uint8_t* smem_b = smem + nst * kABytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + nst * C::stage_bytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + nst;

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const int wg = warp >> 2;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmA[0]);
        tma_prefetch_desc(&p.tmA[1]);
        tma_prefetch_desc(&p.tmB);
        for (int s = 0; s < nst; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2);       // one arrive per consumer warpgroup
        }
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
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = tile0; tile < num_tiles; tile += tile_step) {
            const int m_tile = tile % m_groups, n_tile = tile / m_groups;
            const int x0 = (m_tile % p.tiles_x) * p.tw;
            const int y0 = ((m_tile / p.tiles_x) % p.tiles_y) * p.th;
            const int b0 = (m_tile / (p.tiles_x * p.tiles_y)) * p.tb;
            int kb_global = 0;
            for (int s = 0; s < p.num_segs; ++s) {
                const CUtensorMap* ma = &p.tmA[p.seg_map[s]];
                const int dy = p.seg_dy[s], dx = p.seg_dx[s];
                for (int kb = 0; kb < p.seg_kb[s]; ++kb, ++kb_global) {
                    mbar_wait(&empty[stage], phase ^ 1, p.err_flag, 1);
                    if (elect_one()) {
                        if (tile == tile0 && kb_global < early_kb) {
                            // expect_tx and the weight tile were issued before griddepcontrol.wait
                            tma_load_4d(smem_a + stage * kABytes, ma, &full[stage], kb * kBK, x0 + dx, y0 + dy, b0);
                        } else {
                            mbar_expect_tx(&full[stage], C::stage_bytes);
                            tma_load_4d(smem_a + stage * kABytes, ma, &full[stage], kb * kBK, x0 + dx, y0 + dy, b0);
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

    // ===================== consumers: warpgroup 1 rows [0,64), warpgroup 2 rows [64,128) of the tile =====================
    reg_alloc<232>();
    const int cw = wg - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int quad = lane & 3;
    int rr[2], ww[2], hh[2], bb[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        rr[i] = cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;      // accumulator row inside the 128-row tile
        ww[i] = rr[i] % p.tw;
        hh[i] = (rr[i] / p.tw) % p.th;
        bb[i] = rr[i] / (p.tw * p.th);
    }
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
        const int m_tile = tile % m_groups, n_tile = tile / m_groups;
        bool row_ok[2];
        long long row[2];
        int bidx[2];
        float ln_mu[2] = {0.f, 0.f}, ln_rstd[2] = {1.f, 1.f};
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int x = (m_tile % p.tiles_x) * p.tw + ww[i];
            const int y = ((m_tile / p.tiles_x) % p.tiles_y) * p.th + hh[i];
            const int b = (m_tile / (p.tiles_x * p.tiles_y)) * p.tb + bb[i];
            row_ok[i] = (x < p.W) && (y < p.H) && (b < p.B);
            row[i] = ((long long)b * p.H + y) * p.W + x;
            bidx[i] = b;
            if (p.ln_stats) ln_row_stats(p, row[i], row_ok[i], ln_mu[i], ln_rstd[i]);
        }
        // ---- main loop: one k-block of wgmmas in flight; the slot of the previous k-block is released once done
        int prev_stage = -1;
        for (int kb = 0; kb < p.total_kb; ++kb) {
            mbar_wait(&full[stage], phase, p.err_flag, 3);
            const uint32_t a_addr = smem_u32(smem_a + stage * kABytes) + cw * (64 * 128);
            const uint32_t b_addr = smem_u32(smem_b + stage * C::b_bytes);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBK / 16; ++k)
                WgmmaSS<BN>::template mma<0>(acc, make_smem_desc_sw128(a_addr + k * 32, 16, 1024),
                                             make_smem_desc_sw128(b_addr + k * 32, 16, 1024), (kb | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            fence_regs(acc);
            if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);
            prev_stage = stage;
            if (++stage == nst) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);

        // ---- epilogue from registers: this thread holds rows rr[0], rr[1] and columns 8j + 2*quad + {0, 1}
        if (p.mode == 0) {
            const int n_base = n_tile * BN + 2 * quad;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float st_sum = 0.f, st_sq = 0.f;
                if (row_ok[i]) {
                    const __half* res_row = p.res ? p.res + row[i] * p.ldr : nullptr;
                    __half* out_row = p.out + row[i] * p.ldo;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j) {
                        const int n = n_base + 8 * j;
                        if (n < p.N) {        // N is a multiple of 8 (checked on the host)
                            float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
                            if (p.ln_stats) {
                                const float2 c = ld_f2(p.ln_csum + n), t = ld_f2(p.ln_bias + n);
                                v0 = fmaf(ln_rstd[i], v0 - ln_mu[i] * c.x, t.x);
                                v1 = fmaf(ln_rstd[i], v1 - ln_mu[i] * c.y, t.y);
                            } else if (p.bias) {
                                const float2 t = ld_h2(p.bias + n);
                                v0 += t.x;
                                v1 += t.y;
                            }
                            if (p.bias2) {
                                const float2 t = ld_h2(p.bias2 + (long long)bidx[i] * p.bias2_ld + n);
                                v0 += t.x;
                                v1 += t.y;
                            }
                            if (res_row) {
                                const float2 t = __half22float2(*reinterpret_cast<const __half2*>(res_row + n));
                                v0 += t.x;
                                v1 += t.y;
                            }
                            if (p.relu) {
                                v0 = fmaxf(v0, 0.f);
                                v1 = fmaxf(v1, 0.f);
                            }
                            const __half2 o = __floats2half2_rn(v0, v1);
                            *reinterpret_cast<__half2*>(out_row + n) = o;
                            if (p.stats_out) {       // statistics of the STORED (fp16-rounded) values
                                const float2 f = __half22float2(o);
                                st_sum += f.x + f.y;
                                st_sq = fmaf(f.x, f.x, fmaf(f.y, f.y, st_sq));
                            }
                        }
                    }
                    if (p.stats_out)
                        p.stats_out[row[i] * (kEpiParts * p.tiles_n) + kEpiParts * n_tile + quad] =
                            make_float2(st_sum, st_sq);
                }
            }
        } else {
            // GEGLU: tile columns [0,BN/2) are "value", [BN/2,BN) the matching "gate" (weights are
            // row-interleaved per tile on the host); out = (v+bv) * gelu(g+bg), BN/2 outputs per tile.
            constexpr int HN = BN / 2;
            const int o_base = n_tile * HN + 2 * quad;     // output column base
            const int a_base = n_tile * BN + 2 * quad;     // accumulator (bias) column base
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                if (!row_ok[i]) continue;
                __half* out_row = p.out + row[i] * p.ldo;
#pragma unroll
                for (int j = 0; j < HN / 8; ++j) {
                    float v[2] = {acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]};
                    float g[2] = {acc[4 * (j + HN / 8) + 2 * i], acc[4 * (j + HN / 8) + 2 * i + 1]};
                    float2 bv = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
                    if (p.ln_stats) {
                        const float2 cv = ld_f2(p.ln_csum + a_base + 8 * j), cg = ld_f2(p.ln_csum + a_base + HN + 8 * j);
                        bv = ld_f2(p.ln_bias + a_base + 8 * j);
                        bg = ld_f2(p.ln_bias + a_base + HN + 8 * j);
                        v[0] = ln_rstd[i] * (v[0] - ln_mu[i] * cv.x);
                        v[1] = ln_rstd[i] * (v[1] - ln_mu[i] * cv.y);
                        g[0] = ln_rstd[i] * (g[0] - ln_mu[i] * cg.x);
                        g[1] = ln_rstd[i] * (g[1] - ln_mu[i] * cg.y);
                    } else if (p.bias) {
                        bv = ld_h2(p.bias + a_base + 8 * j);
                        bg = ld_h2(p.bias + a_base + HN + 8 * j);
                    }
                    // the reference rounds proj output, gelu(gate) and the product to fp16
                    const float r0 = lb_round_h(v[0] + bv.x) * lb_round_h(gelu_erf(lb_round_h(g[0] + bg.x)));
                    const float r1 = lb_round_h(v[1] + bv.y) * lb_round_h(gelu_erf(lb_round_h(g[1] + bg.y)));
                    *reinterpret_cast<__half2*>(out_row + o_base + 8 * j) = __floats2half2_rn(r0, r1);
                }
            }
        }
    }
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

// 4-D NHWC activation map: dims (C, W, H, B), box (64, tw, th, tb), 128B swizzle, zero OOB fill.
int encode_act_map(lb_ctx* ctx, CUtensorMap* m, const void* base, int64_t ld, int C, int W, int H, int B, int tw,
                   int th, int tb) {
    EncodeTiledFn enc;
    if (int e = get_encode(ctx, &enc)) return e;
    LB_REQUIRE(lb_aligned16(base), "activation base must be 16-byte aligned");
    LB_REQUIRE(ld % 8 == 0 && ld >= C, "activation row stride must be a multiple of 8 elements and >= C");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * W, (cuuint64_t)ld * 2 * W * H};
    cuuint32_t box[4] = {(cuuint32_t)kBK, (cuuint32_t)tw, (cuuint32_t)th, (cuuint32_t)tb};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(activation C=%d W=%d H=%d B=%d ld=%lld box=%d,%d,%d) failed: %d",
               C, W, H, B, (long long)ld, tw, th, tb, (int)r);
    return 0;
}

int encode_weight_map(lb_ctx* ctx, CUtensorMap* m, const void* base, int64_t ld, int64_t K, int N, int bn) {
    EncodeTiledFn enc;
    if (int e = get_encode(ctx, &enc)) return e;
    LB_REQUIRE(lb_aligned16(base), "weight base must be 16-byte aligned");
    LB_REQUIRE(ld % 8 == 0 && ld >= K, "weight row stride must be a multiple of 8 elements and >= K");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)bn};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weight K=%lld N=%d bn=%d) failed: %d", (long long)K, N, bn,
               (int)r);
    return 0;
}

bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

template <int BN> int launch_bn(const GemmPlan& plan, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        LB_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           Cfg<BN>::smem_bytes(Cfg<BN>::deep)));
        attr_set = true;
    }
    LB_CHECK_CUDA(lb_launch_pdl(gemm_tc_kernel<BN>, dim3((unsigned)plan.grid), dim3(kThreadsGemm),
                                (size_t)Cfg<BN>::smem_bytes(plan.p.stages), st, plan.p));
    return 0;
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
    // --- M tiling: a 128-row tile is a (tw x th x tb) box of pixels
    int tw, th, tb;
    if (d.W >= kBM || (d.H == 1 && d.B == 1)) {   // rows of a plain matrix: ragged tail is zero-filled by TMA
        tw = kBM; th = 1; tb = 1;
    } else {
        LB_REQUIRE(is_pow2(d.W), "gemm: W (%d) < 128 must be a power of two", d.W);
        tw = d.W;
        th = kBM / tw;
        if (th > d.H) {
            LB_REQUIRE(is_pow2(d.H), "gemm: H (%d) must be a power of two when H*W < 128", d.H);
            th = d.H;
        }
        tb = kBM / (tw * th);
    }
    p.tw = tw; p.th = th; p.tb = tb;
    p.W = d.W; p.H = d.H; p.B = d.B;
    p.tiles_x = (int)lb_ceil_div(d.W, tw);
    p.tiles_y = (int)lb_ceil_div(d.H, th);
    const int tiles_b = (int)lb_ceil_div(d.B, tb);
    p.tiles_m = p.tiles_x * p.tiles_y * tiles_b;
    // --- N tiling
    int bn;
    if ((d.mode & 0xff) == 1) {
        bn = (d.mode & LB_GEMM_GEGLU256) ? 256 : 128;      // the weight rows are interleaved per N tile by the caller
        LB_REQUIRE(d.N % bn == 0, "gemm: GEGLU needs N %% %d == 0 (got %d)", bn, d.N);
    } else if (d.N % 256 == 0 && (int64_t)p.tiles_m * (d.N / 256) >= 2 * ctx->sm_count) bn = 256;
    else if (d.N % 160 == 0) bn = 160;
    else if (d.N % 128 == 0) bn = 128;
    else if (d.N <= 64) bn = 64;
    else bn = 128;
    plan->bn = bn;
    p.tiles_n = (int)lb_ceil_div(d.N, bn);
    p.N = d.N;
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
    if (int e = encode_act_map(ctx, &p.tmA[0], d.a0, d.a0_ld, d.a0_c, d.W, d.H, d.B, tw, th, tb)) return e;
    if (d.a1) {
        if (int e = encode_act_map(ctx, &p.tmA[1], d.a1, d.a1_ld, d.a1_c, d.W, d.H, d.B, tw, th, tb)) return e;
    } else {
        p.tmA[1] = p.tmA[0];
    }
    if (int e = encode_weight_map(ctx, &p.tmB, d.w, d.w_ld, Ktot, d.N, bn)) return e;
    p.out = static_cast<__half*>(d.out);
    p.ldo = d.out_ld;
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
    // ring depth: as many stages as 227 KB of shared memory hold (one CTA per SM)
    p.stages = (bn <= 64) ? 8 : (bn <= 128) ? 7 : (bn <= 160) ? 6 : 4;
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
