// program.cu -- the UNet graph executor: a flat, pre-validated list of kernel launches.
//
// The host side (latentblending_b200/unet.py) lowers one SDXL-UNet forward for a fixed
// (batch, height, width) into ~1.7k lb_op records over static device buffers; this file
// turns them into prepared launches once (TMA descriptors encoded, tilings chosen) and
// replays them on a stream with no Python, no allocation and no host sync in the loop.
// Replaces the eager PyTorch module walk behind pipe.unet(...) (diffusers_holder.py:336-344).
#include <stddef.h>
#include <stdlib.h>

#include <vector>

#include "gemm_sm90.cuh"

// the op records are an ABI: a member may grow only inside the union's existing size (set by lb_gemm_desc)
static_assert(sizeof(((lb_op*)nullptr)->u.resample) <= sizeof(lb_gemm_desc), "lb_op.u.resample outgrew the union");
static_assert(sizeof(((lb_op*)nullptr)->u.conv) <= sizeof(lb_gemm_desc), "lb_op.u.conv outgrew the union");
// lb_op.dtype took the place of a reserved int32: the record size and the union's offset are unchanged
static_assert(sizeof(lb_op) == 8 + sizeof(lb_gemm_desc) && offsetof(lb_op, u) == 8, "lb_op layout changed");

struct AttnPlan;
int attn_plan_build_opaque(lb_ctx* ctx, const lb_attn_desc& d, void** plan_out);
int attn_plan_launch_opaque(void* plan, cudaStream_t st);
void attn_plan_free_opaque(void* plan);

int lb_embed_inputs_src(lb_ctx* ctx, float t, const float* t_dev, const void* text_embeds, const void* time_ids, int B,
                        int dim_t, int pooled, int dim_a, void* temb_in, void* add_in, void* stream);
int lb_set_scalar(float* dst_dev, float v, cudaStream_t st);

// Replay mode.  The op list is static, so after one warm (direct) run the whole program is captured ONCE into a CUDA
// graph -- every launch keeps its programmatic-dependent-launch edge -- and later runs are a single cudaGraphLaunch:
// ~700-900 driver launches per UNet forward (2-4 ms of host time) become one, and the device's front end walks a
// pre-built launch list.  The only run-time parameter, the timestep, lives in device memory (t_dev, allocated when a
// capture is first attempted: only the graph reads it).  If capture is not possible (another capture in flight, an
// unsupported driver) the program keeps launching directly.
struct lb_program {
    lb_ctx* ctx;
    struct Node {
        lb_op op;
        GemmPlan gemm;
        void* attn;
    };
    std::vector<Node> nodes;
    float* t_dev = nullptr;
    cudaStream_t capture_stream = nullptr;   // private: the caller's stream may be the legacy default stream, which cannot capture
    cudaGraphExec_t graph_exec = nullptr;
    int runs = 0;
    int graph_state = 0;      // 0 not tried, 1 captured, -1 unavailable
};

// the kinds whose entry point takes a dtype argument (lb_op.dtype); every other kind needs dtype 0
static bool kind_has_dtype(int kind) {
    switch (kind) {
        case LB_OP_GROUPNORM: case LB_OP_LATENT_PREP: case LB_OP_CONV_IN: case LB_OP_UPSAMPLE_NEAREST:
        case LB_OP_NHWC_TO_NCHW: case LB_OP_POSTPROCESS_U8: case LB_OP_SOFTMAX_ROWS:
            return true;
        default:
            return false;
    }
}

static bool lb_graphs_enabled() {
    static int v = -1;
    if (v < 0) v = getenv("LB_NO_GRAPH") ? 0 : 1;
    return v != 0;
}

extern "C" int lb_program_create(lb_ctx* ctx, const lb_op* ops, int64_t n_ops, lb_program** out) {
    LB_REQUIRE(ctx && ops && out && n_ops >= 0, "lb_program_create: bad arguments");
    lb_program* prog = new lb_program();
    prog->ctx = ctx;
    prog->nodes.resize((size_t)n_ops);
    for (int64_t i = 0; i < n_ops; ++i) {
        lb_program::Node& nd = prog->nodes[(size_t)i];
        nd.op = ops[i];
        nd.attn = nullptr;
        int e = 0;
        if (kind_has_dtype(ops[i].kind)) {
            if (ops[i].dtype != LB_DTYPE_F16 && ops[i].dtype != LB_DTYPE_BF16) {
                lb_set_error("lb_program_create: op %lld has unknown dtype %d", (long long)i, ops[i].dtype);
                e = 2;
            }
        } else if (ops[i].dtype != LB_DTYPE_F16) {
            lb_set_error("lb_program_create: op %lld (kind %d) has no dtype %d variant (a GEMM takes its types "
                         "from its mode flags)", (long long)i, ops[i].kind, ops[i].dtype);
            e = 2;
        }
        if (!e) switch (ops[i].kind) {
            case LB_OP_GEMM:
                e = gemm_plan_build(ctx, *reinterpret_cast<const GemmDesc*>(&ops[i].u.gemm), &nd.gemm);
                break;
            case LB_OP_ATTENTION:
                e = attn_plan_build_opaque(ctx, ops[i].u.attn, &nd.attn);
                break;
            case LB_OP_EMBED_INPUTS: case LB_OP_LINEAR_SMALL: case LB_OP_CONV_OUT:
            case LB_OP_UPSAMPLE_NEAREST: case LB_OP_IM2COL_S2: case LB_OP_GROUPNORM: case LB_OP_LAYERNORM:
            case LB_OP_LATENT_PREP: case LB_OP_SOFTMAX_ROWS: case LB_OP_POSTPROCESS_U8:
            case LB_OP_LPIPS_IM2COL_U8: case LB_OP_IM2COL: case LB_OP_MAXPOOL3S2: case LB_OP_NHWC_TO_NCHW:
                break;
            case LB_OP_CONV_IN: {
                const auto& a = ops[i].u.conv;
                if (a.act != 0 && a.act != 1) {
                    lb_set_error("lb_program_create: op %lld: unknown conv_in act %d", (long long)i, a.act);
                    e = 2;
                } else if (a.act == 1 && ops[i].dtype != LB_DTYPE_F16) {
                    lb_set_error("lb_program_create: op %lld: the tiny VAE input stage is fp16-only", (long long)i);
                    e = 2;
                }
                break;
            }
            default:
                lb_set_error("lb_program_create: op %lld has unknown kind %d", (long long)i, ops[i].kind);
                e = 2;
        }
        if (e) {
            char msg[1024];
            snprintf(msg, sizeof(msg), "op %lld (kind %d): %s", (long long)i, ops[i].kind, lb_last_error());
            lb_set_error("%s", msg);
            for (auto& n2 : prog->nodes) if (n2.attn) attn_plan_free_opaque(n2.attn);
            delete prog;
            return e;
        }
    }
    *out = prog;
    return 0;
}

extern "C" int lb_program_destroy(lb_program* prog) {
    if (prog) {
        for (auto& nd : prog->nodes) if (nd.attn) attn_plan_free_opaque(nd.attn);
        if (prog->graph_exec) cudaGraphExecDestroy(prog->graph_exec);
        if (prog->capture_stream) cudaStreamDestroy(prog->capture_stream);
        if (prog->t_dev) cudaFree(prog->t_dev);
        delete prog;
    }
    return 0;
}

extern "C" int64_t lb_program_num_launches(lb_program* prog) {
    if (!prog) return -1;
    int64_t n = 0;
    for (auto& nd : prog->nodes) n += (nd.op.kind == LB_OP_GROUPNORM) ? 2 : 1;
    return n;
}

static int program_launch_all(lb_program* prog, float t, const float* t_dev, uint32_t kind_mask, void* stream);

extern "C" int lb_program_run(lb_program* prog, float t, void* stream) {
    LB_REQUIRE(prog != nullptr, "lb_program_run: null program");
    cudaStream_t st = lb_stream(stream);
    if (!lb_graphs_enabled() || prog->graph_state < 0 || prog->nodes.size() < 8)
        return program_launch_all(prog, t, nullptr, 0xFFFFFFFFu, stream);
    if (prog->graph_state == 0) {
        if (prog->runs++ == 0)                       // first run direct: function attributes get set outside a capture
            return program_launch_all(prog, t, nullptr, 0xFFFFFFFFu, stream);
        cudaGraph_t graph = nullptr;
        int e = 1;
        if (prog->t_dev == nullptr && cudaMalloc(&prog->t_dev, sizeof(float)) != cudaSuccess) prog->t_dev = nullptr;
        if (prog->capture_stream == nullptr &&
            cudaStreamCreateWithFlags(&prog->capture_stream, cudaStreamNonBlocking) != cudaSuccess)
            prog->capture_stream = nullptr;
        if (prog->t_dev != nullptr && prog->capture_stream != nullptr &&
            cudaStreamBeginCapture(prog->capture_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            // nothing executes during capture: the launches only record the node list (with their PDL edges)
            e = program_launch_all(prog, t, prog->t_dev, 0xFFFFFFFFu, prog->capture_stream);
            cudaError_t ce = cudaStreamEndCapture(prog->capture_stream, &graph);
            if (e == 0 && ce == cudaSuccess && graph != nullptr &&
                cudaGraphInstantiate(&prog->graph_exec, graph, 0) == cudaSuccess)
                prog->graph_state = 1;
            if (graph) cudaGraphDestroy(graph);
        }
        if (prog->graph_state != 1) {
            cudaGetLastError();                       // clear the capture error: replay stays on direct launches
            prog->graph_state = -1;
            prog->graph_exec = nullptr;
            return program_launch_all(prog, t, nullptr, 0xFFFFFFFFu, stream);
        }
    }
    if (int e = lb_set_scalar(prog->t_dev, t, st)) return e;
    LB_CHECK_CUDA(cudaGraphLaunch(prog->graph_exec, st));
    return 0;
}

extern "C" int lb_program_is_graph(lb_program* prog) { return prog ? prog->graph_state : -2; }

extern "C" int64_t lb_program_count_kinds(lb_program* prog, uint32_t kind_mask) {
    if (!prog) return -1;
    int64_t n = 0;
    for (auto& nd : prog->nodes)
        if (kind_mask & (1u << nd.op.kind)) n += (nd.op.kind == LB_OP_GROUPNORM) ? 2 : 1;
    return n;
}

extern "C" int lb_program_run_kinds(lb_program* prog, float t, uint32_t kind_mask, void* stream) {
    LB_REQUIRE(prog != nullptr, "lb_program_run: null program");
    return program_launch_all(prog, t, nullptr, kind_mask, stream);
}

static int program_launch_all(lb_program* prog, float t, const float* t_dev, uint32_t kind_mask, void* stream) {
    lb_ctx* ctx = prog->ctx;
    cudaStream_t st = lb_stream(stream);
    for (size_t i = 0; i < prog->nodes.size(); ++i) {
        lb_program::Node& nd = prog->nodes[i];
        const lb_op& o = nd.op;
        if (!(kind_mask & (1u << o.kind))) continue;
        int e = 0;
        switch (o.kind) {
            case LB_OP_GEMM: e = gemm_plan_launch(nd.gemm, st); break;
            case LB_OP_ATTENTION: e = attn_plan_launch_opaque(nd.attn, st); break;
            case LB_OP_EMBED_INPUTS: {
                const auto& a = o.u.embed;
                e = lb_embed_inputs_src(ctx, t, t_dev, a.text_embeds, a.time_ids, a.B, a.dim_t, a.pooled, a.dim_a,
                                        a.temb_in, a.add_in, stream);
                break;
            }
            case LB_OP_LINEAR_SMALL: {
                const auto& a = o.u.lin;
                e = lb_linear_small(ctx, a.x, a.ldx, a.M, a.K, a.w, a.ldw, a.bias, a.addend, a.ldadd, a.act_in,
                                    a.act_out, a.out, a.ldo, a.N, stream);
                break;
            }
            case LB_OP_CONV_IN: {
                const auto& a = o.u.conv;
                e = lb_conv_in(ctx, a.x, a.B, a.Cin, a.H, a.W, a.w, a.bias, a.Cout, a.out, a.ld_out, a.act, a.in_scale,
                               stream, o.dtype);
                break;
            }
            case LB_OP_CONV_OUT: {
                const auto& a = o.u.conv;
                e = lb_conv_out(ctx, a.x, a.ld_x, a.B, a.Cin, a.H, a.W, a.w, a.bias, a.Cout, a.out, stream);
                break;
            }
            case LB_OP_UPSAMPLE_NEAREST: {
                const auto& a = o.u.resample;
                e = lb_upsample_nearest(ctx, a.x, a.ld_x, a.B, a.H, a.W, a.C, a.out, a.ld_out, a.Ho, a.Wo, stream,
                                        o.dtype);
                break;
            }
            case LB_OP_IM2COL_S2: {
                const auto& a = o.u.resample;
                e = lb_im2col_s2(ctx, a.x, a.ld_x, a.B, a.H, a.W, a.C, a.out, stream);
                break;
            }
            case LB_OP_GROUPNORM: {
                const auto& a = o.u.norm;
                e = lb_groupnorm(ctx, a.x, a.ld_x, a.B, (int)a.rows, a.C, a.groups, a.gamma, a.beta, a.eps, a.silu,
                                 a.out, a.ld_out, a.workspace, stream, o.dtype);
                break;
            }
            case LB_OP_LAYERNORM: {
                const auto& a = o.u.norm;
                e = lb_layernorm(ctx, a.x, a.ld_x, a.rows, a.C, a.gamma, a.beta, a.eps, a.out, a.ld_out, stream);
                break;
            }
            case LB_OP_LATENT_PREP: {
                const auto& a = o.u.aux;
                e = lb_latent_prep(ctx, a.x, a.B, a.C, a.n, a.w, a.bias, a.out, stream, o.dtype);
                break;
            }
            case LB_OP_SOFTMAX_ROWS: {
                const auto& a = o.u.aux;
                e = lb_softmax_rows(ctx, a.x, a.ld_x, a.n, a.C, a.out, a.ld_out, stream, o.dtype);
                break;
            }
            case LB_OP_POSTPROCESS_U8: {
                const auto& a = o.u.aux;
                e = lb_postprocess_u8(ctx, a.x, a.B, a.C, a.n, a.out, (int*)const_cast<void*>(a.w), stream, o.dtype);
                break;
            }
            case LB_OP_NHWC_TO_NCHW: {
                const auto& a = o.u.aux;
                e = lb_nhwc_to_nchw(ctx, a.x, a.ld_x, a.B, a.C, a.n, a.out, stream, o.dtype);
                break;
            }
            case LB_OP_LPIPS_IM2COL_U8: {
                const auto& a = o.u.patch;
                e = lb_lpips_im2col_u8(ctx, a.x, a.H, a.W, a.k, a.stride, a.pad, a.f, a.f + 3, a.out, a.C, stream);
                break;
            }
            case LB_OP_IM2COL: {
                const auto& a = o.u.patch;
                e = lb_im2col(ctx, a.x, a.ld_x, a.H, a.W, a.C, a.k, a.stride, a.pad, a.out, stream);
                break;
            }
            case LB_OP_MAXPOOL3S2: {
                const auto& a = o.u.patch;
                e = lb_maxpool3s2(ctx, a.x, a.ld_x, a.H, a.W, a.C, a.out, a.ld_out, stream);
                break;
            }
        }
        if (e) return e;
    }
    return 0;
}
