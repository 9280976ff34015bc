// attn_sm90.cu -- K8: fused softmax(Q K^T / sqrt(d)) V for head dim 64 on wgmma (sm_90a).
//
// Replaces F.scaled_dot_product_attention under diffusers' AttnProcessor2_0 in
// every transformer block of the SDXL UNet (call site
// latentblending/diffusers_holder.py:336-344): self-attention (S = 4096 / 1024,
// Q,K,V slices of one fused-QKV activation) and cross-attention to the 77 text
// tokens (K,V slices of a [B,77,2C] projection).  fp16 in, fp32 softmax, fp16 out.
//
// One CTA = 128 query rows of one (batch, head), three warpgroups:
//   warpgroup 0    TMA producer: the Q tile once, then 128-key K / V tiles into a two-stage ring (128B-swizzled)
//   warpgroups 1-2 64 query rows each, per 128-key tile:
//     S = Q K^T   wgmma m64n128k16 x4, Q and K K-major from shared memory, S in registers (fp32)
//     softmax     online (running row max and row sum per row; the four lanes of a quad share a row), exps on MUFU.EX2
//     O += P V    wgmma m64n64k16 x8 with P as the register A operand (fp16), V consumed MN-major from its TMA tile
//   O is normalised by the row sum once, at the end.
// Bound: tensor pipe / MUFU.EX2.  Algorithmic FLOPs = 4*Sq*Skv*64 per head.
#include <stdlib.h>

#include "common.cuh"
#include "sm90.cuh"

using namespace sm90;

struct alignas(64) AttnParams {
    CUtensorMap tmQ, tmK, tmV;     // 3-D maps (columns, rows, batch), box (64, 128, 1), 128B swizzle
    int Sq, Skv, heads, B;
    int q_col0, k_col0, v_col0;    // column of head 0 inside each buffer
    __half* out; long long ldo;    // [B*Sq, heads*64]
    float scale_log2;              // softmax scale * log2(e)
    int* err_flag;
};

namespace {

constexpr int kD = 64, kBQ = 128, kBKV = 128;   // one CTA: 128 query rows (64 per consumer warpgroup), 128-key tiles
constexpr int kTileBytes = 128 * 64 * 2;        // 16 KiB: the Q tile / one K / V tile
constexpr int kKVStages = 2;
constexpr int kAttnSmem = (1 + 2 * kKVStages) * kTileBytes + 1024 + 256;
constexpr int kAttnThreads = 384;

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

__global__ void __launch_bounds__(kAttnThreads, 1) attn_tc_kernel(const __grid_constant__ AttnParams p) {
    pdl_launch_dependents();
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + kTileBytes;                        // kKVStages
    uint8_t* sV = sK + kKVStages * kTileBytes;            // kKVStages
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kKVStages * kTileBytes);
    uint64_t* q_full = bars + 0;
    uint64_t* k_full = bars + 1;     // [2]
    uint64_t* k_empty = bars + 3;    // [2]
    uint64_t* v_full = bars + 5;     // [2]
    uint64_t* v_empty = bars + 7;    // [2]

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int q0 = blockIdx.x * kBQ, head = blockIdx.y, b = blockIdx.z;
    const int nkv = (p.Skv + kBKV - 1) / kBKV;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmQ);
        tma_prefetch_desc(&p.tmK);
        tma_prefetch_desc(&p.tmV);
        mbar_init(q_full, 1);
        for (int i = 0; i < kKVStages; ++i) {
            mbar_init(&k_full[i], 1);
            mbar_init(&k_empty[i], 2);     // one arrive per consumer warpgroup
            mbar_init(&v_full[i], 1);
            mbar_init(&v_empty[i], 2);
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();

    if (wg == 0) {
        reg_dealloc<40>();
        if (warp != 0) return;
        // ---------------- TMA producer (warp-uniform loop, one elected lane issues) ----------------
        if (elect_one()) {
            mbar_expect_tx(q_full, kTileBytes);
            tma_load_3d(sQ, &p.tmQ, q_full, p.q_col0 + head * kD, q0, b);
        }
        __syncwarp();
        for (int j = 0; j < nkv; ++j) {
            const int st = j & 1;
            const uint32_t ph = (j >> 1) & 1;
            mbar_wait(&k_empty[st], ph ^ 1, p.err_flag, 11);
            if (elect_one()) {
                mbar_expect_tx(&k_full[st], kTileBytes);
                tma_load_3d(sK + st * kTileBytes, &p.tmK, &k_full[st], p.k_col0 + head * kD, j * kBKV, b);
            }
            __syncwarp();
            mbar_wait(&v_empty[st], ph ^ 1, p.err_flag, 12);
            if (elect_one()) {
                mbar_expect_tx(&v_full[st], kTileBytes);
                tma_load_3d(sV + st * kTileBytes, &p.tmV, &v_full[st], p.v_col0 + head * kD, j * kBKV, b);
            }
            __syncwarp();
        }
        return;
    }

    // ---------------- consumers: 64 query rows per warpgroup ----------------
    reg_alloc<232>();
    const int cw = wg - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int quad = lane & 3;
    const uint32_t q_addr = smem_u32(sQ) + cw * (64 * 128), k_addr = smem_u32(sK), v_addr = smem_u32(sV);
    const float sc = p.scale_log2;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // m_run in the scaled (log2) domain
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float s[64];
    mbar_wait(q_full, 0, p.err_flag, 13);
    for (int j = 0; j < nkv; ++j) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        const int kv_valid = min(kBKV, p.Skv - j * kBKV);
        mbar_wait(&k_full[st], ph, p.err_flag, 14);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kD / 16; ++k)
            WgmmaSS<128>::mma<0>(s, make_smem_desc_sw128(q_addr + k * 32, 16, 1024),
                                 make_smem_desc_sw128(k_addr + st * kTileBytes + k * 32, 16, 1024), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
        if (wg_leader) mbar_arrive(&k_empty[st]);
        // s[4c + 2i + e]: row 16*warp + lane/4 + 8i, key column 8c + 2*quad + e
        if (kv_valid < kBKV) {
#pragma unroll
            for (int c = 0; c < 16; ++c)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (8 * c + 2 * quad + e >= kv_valid) s[4 * c + e] = s[4 * c + 2 + e] = -INFINITY;
        }
        float alpha[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float mx = -INFINITY;
#pragma unroll
            for (int c = 0; c < 16; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * i], s[4 * c + 2 * i + 1]));
            const float m_new = fmaxf(m_run[i], quad_max(mx) * sc);
            alpha[i] = ex2_approx(m_run[i] - m_new);                  // first tile: 2^(-inf) = 0
            m_run[i] = m_new;
            float psum = 0.f;
#pragma unroll
            for (int c = 0; c < 16; ++c)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pv = ex2_approx(fmaf(s[4 * c + 2 * i + e], sc, -m_new));
                    s[4 * c + 2 * i + e] = pv;
                    psum += pv;
                }
            l_run[i] = l_run[i] * alpha[i] + psum;
        }
#pragma unroll
        for (int c = 0; c < 8; ++c)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                o[4 * c + 2 * i] *= alpha[i];
                o[4 * c + 2 * i + 1] *= alpha[i];
            }
        // P as the A operand of O += P V: k-step t covers key columns [16t, 16t + 16)
        uint32_t pa[8][4];
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            pa[t][0] = pack_h2(s[8 * t + 0], s[8 * t + 1]);
            pa[t][1] = pack_h2(s[8 * t + 2], s[8 * t + 3]);
            pa[t][2] = pack_h2(s[8 * t + 4], s[8 * t + 5]);
            pa[t][3] = pack_h2(s[8 * t + 6], s[8 * t + 7]);
        }
        mbar_wait(&v_full[st], ph, p.err_flag, 16);
        fence_regs(o);
        wgmma_fence();
#pragma unroll
        for (int t = 0; t < 8; ++t)
            WgmmaRS<64>::mma<1>(o, pa[t], make_smem_desc_sw128(v_addr + st * kTileBytes + t * 2048, 8192, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o);
        if (wg_leader) mbar_arrive(&v_empty[st]);
    }
    // ---- output O / l: this thread holds rows 16*warp + lane/4 + 8i, columns 8c + 2*quad + e
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int q = q0 + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
        const float inv = 1.0f / quad_sum(l_run[i]);
        if (q < p.Sq) {
            __half* dst = p.out + ((long long)b * p.Sq + q) * p.ldo + head * kD + 2 * quad;
#pragma unroll
            for (int c = 0; c < 8; ++c)
                *reinterpret_cast<__half2*>(dst + 8 * c) = __floats2half2_rn(o[4 * c + 2 * i] * inv, o[4 * c + 2 * i + 1] * inv);
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_rows_map(lb_ctx* ctx, CUtensorMap* m, const void* base, int64_t ld, int64_t cols, int rows, int B) {
    if (!ctx->tmap_encode) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qres;
        LB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres));
        LB_REQUIRE(f != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
        ctx->tmap_encode = f;
    }
    EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(ctx->tmap_encode);
    LB_REQUIRE(lb_aligned16(base) && ld % 8 == 0 && cols <= ld, "attention: operand alignment / stride");
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * rows};
    cuuint32_t box[3] = {64, 128, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(attention cols=%lld rows=%d B=%d) failed: %d",
               (long long)cols, rows, B, (int)r);
    return 0;
}

}  // namespace

int* lb_err_flag(lb_ctx* ctx);

struct AttnPlan {
    AttnParams p;
    dim3 grid;
};

int attn_plan_build(lb_ctx* ctx, const lb_attn_desc& d, AttnPlan* plan) {
    LB_REQUIRE(ctx && plan, "attention: null ctx/plan");
    LB_REQUIRE(d.q && d.k && d.v && d.out, "attention: null buffer");
    LB_REQUIRE(d.head_dim == 64, "attention: only head_dim 64 is implemented (got %d)", d.head_dim);
    LB_REQUIRE(d.B >= 1 && d.heads >= 1 && d.Sq >= 1 && d.Skv >= 1, "attention: bad sizes");
    LB_REQUIRE(d.out_ld % 8 == 0 && lb_aligned16(d.out), "attention: out alignment");
    AttnParams& p = plan->p;
    memset(&p, 0, sizeof(p));
    const int width = d.heads * 64;
    if (int e = encode_rows_map(ctx, &p.tmQ, d.q, d.q_ld, d.q_col0 + width, d.Sq, d.B)) return e;
    if (int e = encode_rows_map(ctx, &p.tmK, d.k, d.k_ld, d.k_col0 + width, d.Skv, d.B)) return e;
    if (int e = encode_rows_map(ctx, &p.tmV, d.v, d.v_ld, d.v_col0 + width, d.Skv, d.B)) return e;
    p.Sq = d.Sq; p.Skv = d.Skv; p.heads = d.heads; p.B = d.B;
    p.q_col0 = d.q_col0; p.k_col0 = d.k_col0; p.v_col0 = d.v_col0;
    p.out = static_cast<__half*>(d.out);
    p.ldo = d.out_ld;
    p.scale_log2 = d.scale * 1.4426950408889634f;
    p.err_flag = lb_err_flag(ctx);
    plan->grid = dim3((unsigned)lb_ceil_div(d.Sq, kBQ), (unsigned)d.heads, (unsigned)d.B);
    return 0;
}

int attn_plan_launch(const AttnPlan& plan, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        LB_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem));
        attr_set = true;
    }
    lb_launch_pdl(attn_tc_kernel, plan.grid, dim3(kAttnThreads), (size_t)kAttnSmem, st, plan.p);
    LB_LAUNCH_CHECK();
    return 0;
}

extern "C" int lb_attention(lb_ctx* ctx, const lb_attn_desc* desc, void* stream) {
    LB_REQUIRE(ctx && desc, "lb_attention: null argument");
    AttnPlan plan;
    if (int e = attn_plan_build(ctx, *desc, &plan)) return e;
    return attn_plan_launch(plan, lb_stream(stream));
}

// opaque handles for program.cu (AttnPlan holds CUtensorMaps and needs 64-byte alignment)
int attn_plan_build_opaque(lb_ctx* ctx, const lb_attn_desc& d, void** plan_out) {
    AttnPlan* plan = new AttnPlan();
    if (int e = attn_plan_build(ctx, d, plan)) {
        delete plan;
        return e;
    }
    *plan_out = plan;
    return 0;
}
int attn_plan_launch_opaque(void* plan, cudaStream_t st) { return attn_plan_launch(*static_cast<AttnPlan*>(plan), st); }
void attn_plan_free_opaque(void* plan) { delete static_cast<AttnPlan*>(plan); }
