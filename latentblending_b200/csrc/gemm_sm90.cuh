// gemm_sm90.cuh -- host-side plan object of the wgmma GEMM / implicit-GEMM conv kernel (K7 + K4).
#pragma once
#include "common.cuh"

// Mirrors lb_gemm_desc of include/lb200.h (kept in sync by hand; plain C layout).
struct GemmDesc {
    const void* a0; int64_t a0_ld; int32_t a0_c;
    const void* a1; int64_t a1_ld; int32_t a1_c;
    int32_t B, H, W;
    int32_t taps;
    const void* w; int64_t w_ld;
    int32_t N;
    const void* bias;
    const void* bias2; int64_t bias2_ld;
    const void* res; int64_t res_ld;
    void* out; int64_t out_ld;
    int32_t mode;   // low byte: 0 linear epilogue, 1 GEGLU (N accumulators -> N/2 outputs); | LB_GEMM_STATIC_W | LB_GEMM_RELU
                    // | LB_GEMM_TILE_BOX | LB_GEMM_TILE_RUNS | LB_GEMM_BF16 | LB_GEMM_OUT_F16 | LB_GEMM_D2S2
};

constexpr int kGemmMaxSegs = 12;

struct alignas(64) GemmParams {
    CUtensorMap tmA[2];
    CUtensorMap tmB;
    int num_segs;
    int seg_map[kGemmMaxSegs], seg_dy[kGemmMaxSegs], seg_dx[kGemmMaxSegs], seg_kb[kGemmMaxSegs];
    int total_kb;
    int W, H, B;
    int tw, th, tb;        // pixel-box tiling: a tile is a (tw x th x tb) box, tiles_x * tiles_y * ceil(B / tb) of them
    int tiles_x, tiles_y, tiles_m, tiles_n;
    int N;
    int mode;
    int static_w;  // weights may be fetched before griddepcontrol.wait (LB_GEMM_STATIC_W)
    // fp16, or bf16 in the bf16 instantiations (LB_GEMM_BF16), which reinterpret these pointers
    __half* out; long long ldo;
    const __half* bias;
    const __half* bias2; long long bias2_ld;
    const __half* res; long long ldr;
    int* err_flag;
    int relu;      // mode 0: out = max(out, 0) (LB_GEMM_RELU)
    // pixel-run tiling (runs = 1): tile m is rows [128 m, 128 m + 128) of the flattened b*H*W + y*W + x pixel order
    // (it may span image rows and images; M = B*H*W < 2^31), loaded by TMA im2col runs
    int runs;
    int M, HW;
    int out_f16;   // bf16 instantiations: the output is stored as fp16 (LB_GEMM_OUT_F16)
    int d2s_co;    // depth-to-space kernels (LB_GEMM_D2S2): output channels per phase, N / 4
};

struct GemmPlan {
    GemmParams p;
    int bn;        // N tile: 64 / 128 / 160 / 256
    bool bf16;     // operands, bias, residual (and, unless p.out_f16, the output) are bf16
    bool d2s;      // LB_GEMM_D2S2: the depth-to-space kernels
    int grid;
};

int gemm_plan_build(lb_ctx* ctx, const GemmDesc& d, GemmPlan* plan);
int gemm_plan_launch(const GemmPlan& plan, cudaStream_t st);
int* lb_err_flag(lb_ctx* ctx);
