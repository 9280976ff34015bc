// common.cuh -- shared host/device helpers for liblb200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/lb200.h"

struct lb_ctx {
    int device;
    int sm_count;
    int smem_optin;       // max dynamic smem per block (bytes)
    void* tmap_encode;    // cuTensorMapEncodeTiled, resolved lazily through the runtime
    void* tmap_encode_im2col;   // cuTensorMapEncodeIm2col, likewise
    int* err_flag_dev;    // protocol-error code written by a kernel before it traps
};

// ---- error plumbing ---------------------------------------------------------
void lb_set_error(const char* fmt, ...);

#define LB_CHECK_CUDA(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            lb_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,              \
                         cudaGetErrorString(_e));                                        \
            return 1;                                                                    \
        }                                                                                \
    } while (0)

#define LB_REQUIRE(cond, ...)                                                            \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            lb_set_error(__VA_ARGS__);                                                   \
            return 2;                                                                    \
        }                                                                                \
    } while (0)

#define LB_LAUNCH_CHECK()                                                                \
    do {                                                                                 \
        cudaError_t _e = cudaGetLastError();                                             \
        if (_e != cudaSuccess) {                                                         \
            lb_set_error("%s:%d: kernel launch failed: %s", __FILE__, __LINE__,          \
                         cudaGetErrorString(_e));                                        \
            return 1;                                                                    \
        }                                                                                \
    } while (0)

static inline cudaStream_t lb_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline bool lb_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline int64_t lb_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- launches: programmatic dependent launch (PDL) ---------------------------------------------
// Every kernel of the library is launched with programmatic stream serialization and starts with
// griddepcontrol.launch_dependents / griddepcontrol.wait: the NEXT kernel's launch latency, block scheduling and
// prologue (barrier init, descriptor prefetch) overlap this kernel's execution; its
// griddepcontrol.wait returns only when this grid has completed and its writes are visible.
#ifdef __CUDACC__
#include <utility>
bool lb_pdl_enabled();
template <typename... KArgs, typename... Args>
static inline cudaError_t lb_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                        Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = lb_pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

// ---- device helpers ---------------------------------------------------------
#ifdef __CUDACC__
// fp16 rounding of an fp32 value exactly as a torch fp16 op stores it
__device__ __forceinline__ float lb_round_h(float x) { return __half2float(__float2half_rn(x)); }

// The 16-bit storage types of the kernels that exist in fp16 and bf16 (LB_DTYPE_F16 / LB_DTYPE_BF16): the element
// type T, its pair type, and fp32 <-> T conversions.  Both are 2 bytes, so vector widths and strides do not change.
template <typename T> struct LbType;
template <> struct LbType<__half> {
    using T2 = __half2;
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ float2 to_f2(__half2 v) { return __half22float2(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
    static __device__ __forceinline__ __half2 from_f2(float a, float b) { return __floats2half2_rn(a, b); }
    static __device__ __forceinline__ __half2 zero2() { return __float2half2_rn(0.f); }
    static __device__ __forceinline__ float round(float v) { return lb_round_h(v); }
};
template <> struct LbType<__nv_bfloat16> {
    using T2 = __nv_bfloat162;
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ float2 to_f2(__nv_bfloat162 v) { return __bfloat1622float2(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
    static __device__ __forceinline__ __nv_bfloat162 from_f2(float a, float b) { return __floats2bfloat162_rn(a, b); }
    static __device__ __forceinline__ __nv_bfloat162 zero2() { return __float2bfloat162_rn(0.f); }
    static __device__ __forceinline__ float round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
};

// 128-bit streaming load/store (read-once data: do not allocate in L1)
__device__ __forceinline__ uint4 lb_ldg_stream(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void lb_stg_stream(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
}

__device__ __forceinline__ double lb_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float lb_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif
