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

// Philox4x32-10 (Salmon et al., SC'11) on the 128-bit counter (ctr as u64 -> words 0, 1; words 2, 3 = 0) and a 64-bit key
// (tests/augment_ref.py::philox4x32_10 restates it)
__device__ __forceinline__ void philox4x32_10(uint64_t key, uint64_t ctr, uint32_t out[4])
{
    uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
    uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
#pragma unroll
    for (int i = 0; i < 10; i++) {
        if (i) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Saturate to the fp16 range before a float -> half conversion: finite overflow and +-inf go to +-65504, NaN stays NaN
// (fminf / fmaxf alone would return the non-NaN operand and turn a NaN into -65504)
__device__ __forceinline__ float sat_f16(float v) { return v != v ? v : fminf(fmaxf(v, -65504.f), 65504.f); }

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
