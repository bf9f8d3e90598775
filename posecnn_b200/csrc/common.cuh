// common.cuh — shared helpers for the sm_90a kernels behind include/posecnn_b200.h
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/posecnn_b200.h"

namespace pcnn {

void set_error(const char* fmt, ...);
// > 48 KB dynamic shared memory opt-in, once per (kernel, device); returns PCNN_OK or PCNN_E_CUDA (api.cu)
int smem_optin(const void* func, int bytes, const char* what);
#define PCNN_SMEM_OPTIN(kernel, bytes, what)                                        \
    do {                                                                            \
        int rc_ = pcnn::smem_optin((const void*)(kernel), (int)(bytes), what);      \
        if (rc_) return rc_;                                                        \
    } while (0)

inline int check_launch(const char* what)
{
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return PCNN_E_CUDA;
    }
    return PCNN_OK;
}

#define PCNN_REQUIRE(cond, ...)            \
    do {                                   \
        if (!(cond)) {                     \
            pcnn::set_error(__VA_ARGS__);  \
            return PCNN_E_INVALID;         \
        }                                  \
    } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// streaming (read-once) 128-bit load / store: keep L1 for data that is actually reused
__device__ __forceinline__ float4 ld_stream_f4(const float4* p)
{
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, const float4& v)
{
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w));
}

}  // namespace pcnn
