// api.cu -- context and error plumbing of the C ABI (include/lb200.h).
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"

int* lb_err_flag(lb_ctx* ctx);

static thread_local char g_err[1024] = "";

void lb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

bool lb_pdl_enabled() {
    static int v = -1;
    if (v < 0) v = getenv("LB_NO_PDL") ? 0 : 1;
    return v != 0;
}

extern "C" int lb_abi_version(void) { return LB_ABI_VERSION; }
extern "C" const char* lb_last_error(void) { return g_err; }

extern "C" int lb_ctx_create(int device, lb_ctx** out) {
    LB_REQUIRE(out != nullptr, "lb_ctx_create: null out pointer");
    int count = 0;
    LB_CHECK_CUDA(cudaGetDeviceCount(&count));
    LB_REQUIRE(device >= 0 && device < count, "lb_ctx_create: device %d out of range (%d devices)", device, count);
    cudaDeviceProp prop;
    LB_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    LB_REQUIRE(prop.major == 9 && prop.minor == 0, "lb_ctx_create: liblb200 is built for sm_90a only; device %d is sm_%d%d",
               device, prop.major, prop.minor);
    lb_ctx* c = new lb_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->smem_optin = (int)prop.sharedMemPerBlockOptin;
    c->tmap_encode = nullptr;
    c->tmap_encode_im2col = nullptr;
    c->err_flag_dev = nullptr;
    LB_CHECK_CUDA(cudaSetDevice(device));
    LB_CHECK_CUDA(cudaMalloc(&c->err_flag_dev, sizeof(int)));
    LB_CHECK_CUDA(cudaMemset(c->err_flag_dev, 0, sizeof(int)));
    *out = c;
    return 0;
}

int* lb_err_flag(lb_ctx* ctx) { return ctx->err_flag_dev; }

extern "C" int lb_ctx_error_flag(lb_ctx* ctx, int* out_code) {
    LB_REQUIRE(ctx && out_code, "lb_ctx_error_flag: null argument");
    cudaError_t e = cudaMemcpy(out_code, ctx->err_flag_dev, sizeof(int), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) {
        lb_set_error("lb_ctx_error_flag: %s", cudaGetErrorString(e));
        return 1;
    }
    cudaMemset(ctx->err_flag_dev, 0, sizeof(int));
    return 0;
}

extern "C" int lb_ctx_destroy(lb_ctx* ctx) {
    if (ctx && ctx->err_flag_dev) cudaFree(ctx->err_flag_dev);
    delete ctx;
    return 0;
}

extern "C" int lb_ctx_sm_count(lb_ctx* ctx) { return ctx ? ctx->sm_count : -1; }
