// Shared helpers for the sm_90a kernels behind include/sae_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include "../../include/sae_b200.h"

namespace sae {

extern thread_local char g_err[512];
extern std::atomic<int64_t> g_launches;

inline int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SAE_E_CUDA, "%s: launch failed: %s", what, cudaGetErrorString(e));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return SAE_OK;
}

#define SAE_CUDA_TRY(expr)                                                                   \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess)                                                               \
            return ::sae::fail(SAE_E_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,      \
                               cudaGetErrorString(_e));                                      \
    } while (0)

// Device properties are queried once per process (device 0's SM count is representative: one
// process drives one GPU in this design).
int sm_count();

// ---- deterministic mode (the _det entry points) ---------------------------------------------------------------------------
// Every cross-CTA sum is split into slots: each CTA stores its partial with plain stores into a slot-major workspace
// ws[slot][target], and det_reduce adds the slots into the destination in slot order.  Partitions are planned with DET_SMS in
// place of sm_count(), so the order of every addition is a function of the call's arguments alone.
constexpr int DET_SMS = 132;

// workspace regions start on 256-byte boundaries
inline int64_t det_region(int64_t floats) { return (floats * 4 + 255) & ~(int64_t)255; }

// The two-phase workspace protocol: workspace == NULL stores `need` in *workspace_bytes and sets *query; a workspace smaller
// than `need` is refused.  No CUDA call is made either way.
inline int det_workspace(const void* workspace, int64_t* workspace_bytes, int64_t need, const char* who, bool* query) {
    *query = false;
    if (!workspace_bytes) return fail(SAE_E_INVALID, "%s: null workspace_bytes", who);
    if (!workspace) {
        *workspace_bytes = need;
        *query = true;
        return SAE_OK;
    }
    if (*workspace_bytes < need)
        return fail(SAE_E_INVALID, "%s: workspace of %lld bytes, %lld needed", who, (long long)*workspace_bytes, (long long)need);
    return SAE_OK;
}

// dst[i] (+)= sum_{s < slots} ws[s * n + i], slots added in order; accumulate = 0 overwrites dst; round_tf32 rounds the result
int det_reduce(float* dst, const float* ws, int64_t slots, int64_t n, bool accumulate, int round_tf32, cudaStream_t st);

// a drain's contribution: an fp32 atomic into the destination, or (DET) a plain store into the CTA's workspace slot
template <bool DET>
__device__ __forceinline__ void drain_add(float* p, float v) {
    if constexpr (DET) *p = v;
    else atomicAdd(p, v);
}

__device__ __forceinline__ float rna_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}

// split-TF32 ("3xTF32") operand: v ~= hi + lo with hi = rna_tf32(v), lo = rna_tf32(v - hi) (v - hi is exact in fp32), so
// a*b ~= a_hi b_hi + a_hi b_lo + a_lo b_hi on the TF32 tensor cores carries about 22 significant bits per operand
__device__ __forceinline__ void split_tf32(float v, uint32_t& hi, uint32_t& lo) {
    const float h = rna_tf32(v);
    hi = __float_as_uint(h);
    lo = __float_as_uint(rna_tf32(v - h));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

// Epilogue shared by the conv kernels (see sae_conv_epilogue in the header).
struct EpiParams {
    const float* bias;
    const float* noise;
    const float* residual;
    float nw;          // resolved on device from noise_weight pointer
    const float* noise_weight;
    float alpha, gain, res_scale;
    int act, round_tf32;
    uint32_t* act_mask;   // optional: sign bits of the activation output, 1 bit per element (see sae_conv_epilogue)
};

inline EpiParams make_epi(const sae_conv_epilogue* e) {
    EpiParams p;
    p.bias = nullptr; p.noise = nullptr; p.residual = nullptr; p.noise_weight = nullptr;
    p.nw = 0.f; p.alpha = 0.2f; p.gain = 1.f; p.res_scale = 1.f; p.act = 1; p.round_tf32 = 0; p.act_mask = nullptr;
    if (e) {
        p.bias = e->bias; p.noise = e->noise; p.noise_weight = e->noise_weight;
        p.residual = e->residual; p.alpha = e->alpha; p.gain = e->gain;
        p.res_scale = e->res_scale; p.act = e->act; p.round_tf32 = e->round_tf32; p.act_mask = e->act_mask;
    }
    return p;
}

__device__ __forceinline__ float apply_epi(const EpiParams& e, float v, int64_t pixel, int col, int64_t ldc) {
    if (e.bias) v += __ldg(e.bias + col);
    if (e.noise) v += __ldg(e.noise_weight) * __ldg(e.noise + pixel);
    if (e.act == 3) v = (v > 0.f ? v : v * e.alpha);
    v *= e.gain;
    if (e.residual) v = (v + __ldg(e.residual + pixel * ldc + col)) * e.res_scale;
    if (e.round_tf32) v = rna_tf32(v);
    return v;
}

}  // namespace sae
