// Exponential moving average of the encoder and generator weights (SwappingAutoencoderOptimizer with opt.ema_kimg > 0):
// after every G update the shadow copy moves towards the parameters,  shadow = fmaf(beta, shadow - p, p),  with the
// StyleGAN2-ADA schedule (ema_kimg / ema_rampup) evaluated on the device from the update counter, so one captured G graph
// serves every step of the ramp.  The shadow uses the layout of the G group's Adam moments (segments 16-byte aligned).
#include "common.cuh"

namespace sae {

constexpr int EMA_THREADS = 256;
// as ACC_BLOCKS_PER_TENSOR (accumulate.cu): enough blocks that the largest tensor alone keeps every SM streaming; the blocks of
// a small tensor that find no element exit before reading anything
constexpr int EMA_BLOCKS_PER_TENSOR = 256;

// beta = 0.5^(B / max(h, 1e-8)),  h = half_life (or min(half_life, t * B * rampup) with a ramp), formed in fp64 from the
// number t of averaging updates already made and rounded to fp32 once
__device__ __forceinline__ float ema_beta(int64_t t, float batch_images, float half_life_images, float rampup) {
    double h = (double)half_life_images;
    if (rampup > 0.f) h = fmin(h, (double)t * (double)batch_images * (double)rampup);
    return (float)exp2(-(double)batch_images / fmax(h, 1e-8));
}

__device__ __forceinline__ float4 ema4(float beta, float4 s, float4 p) {
    return make_float4(__fmaf_rn(beta, __fsub_rn(s.x, p.x), p.x), __fmaf_rn(beta, __fsub_rn(s.y, p.y), p.y),
                       __fmaf_rn(beta, __fsub_rn(s.z, p.z), p.z), __fmaf_rn(beta, __fsub_rn(s.w, p.w), p.w));
}

// One grid row (blockIdx.y) per tensor, grid-stride over its elements.  When the parameter and its shadow segment are both
// 16-byte aligned (segments always are; a parameter view may not be) the first 4 * (size / 4) elements go as float4, the
// parameter read with a streaming load; the rest, and every element of an unaligned tensor, one by one.  Elementwise and
// without atomics: the result does not depend on the schedule, so deterministic mode needs no twin.
__global__ void __launch_bounds__(EMA_THREADS)
ema_update_kernel(const float* const* __restrict__ p_ptrs, const int64_t* __restrict__ offsets,
                  const int64_t* __restrict__ sizes, float* __restrict__ shadow, const int64_t* __restrict__ updates,
                  float batch_images, float half_life_images, float rampup, const unsigned long long* __restrict__ skip) {
    const int t = blockIdx.y;
    const float* p = p_ptrs[t];
    if (p == nullptr) return;
    const int64_t size = sizes[t];
    const int64_t first = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    if (blockIdx.x * (int64_t)blockDim.x >= size) return;
    if (skip && *skip) return;
    const float beta = ema_beta(*updates, batch_images, half_life_images, rampup);
    float* s = shadow + offsets[t];
    int64_t tail = 0;
    if (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(s)) & 15) == 0) {
        const int64_t n4 = size / 4;
        const float4* p4 = reinterpret_cast<const float4*>(p);
        float4* s4 = reinterpret_cast<float4*>(s);
        int64_t i = first;
        for (; i + stride < n4; i += 2 * stride) {           // two independent float4 pairs in flight per thread
            const float4 v0 = ldg_stream(p4 + i), v1 = ldg_stream(p4 + i + stride);
            const float4 a0 = s4[i], a1 = s4[i + stride];
            s4[i] = ema4(beta, a0, v0);
            s4[i + stride] = ema4(beta, a1, v1);
        }
        if (i < n4) s4[i] = ema4(beta, s4[i], ldg_stream(p4 + i));
        tail = n4 * 4;
    }
    for (int64_t i = tail + first; i < size; i += stride) {
        const float v = __ldg(p + i);
        s[i] = __fmaf_rn(beta, __fsub_rn(s[i], v), v);
    }
}

// after every block of ema_update_kernel has read *updates (stream order), as adam_advance_kernel follows adam_kernel
__global__ void ema_advance_kernel(int64_t* __restrict__ updates, const unsigned long long* __restrict__ skip) {
    if (skip && *skip) return;
    *updates += 1;
}

}  // namespace sae

using namespace sae;

extern "C" int sae_ema_update(const float* const* p_ptrs, const int64_t* offsets, const int64_t* sizes, int n, float* shadow,
                              int64_t total, int64_t* updates, float batch_images, float half_life_images, float rampup,
                              const unsigned long long* skip, void* stream) {
    if (!p_ptrs || !offsets || !sizes || !shadow || !updates || total < 0)
        return fail(SAE_E_INVALID, "ema_update: null pointer or negative total");
    if (n < 0 || n > 65535) return fail(SAE_E_INVALID, "ema_update: n = %d outside [0, 65535]", n);
    // written as !(x > 0) so that a NaN is refused as well
    if (!(half_life_images > 0.f) || !(rampup >= 0.f) || !(batch_images > 0.f))
        return fail(SAE_E_INVALID, "ema_update: needs half_life_images > 0, rampup >= 0 and batch_images > 0");
    cudaStream_t st = (cudaStream_t)stream;
    if (n > 0) {
        dim3 grid(EMA_BLOCKS_PER_TENSOR, (unsigned)n);
        ema_update_kernel<<<grid, EMA_THREADS, 0, st>>>(p_ptrs, offsets, sizes, shadow, updates, batch_images, half_life_images,
                                                        rampup, skip);
        int rc = check_launch("ema_update");
        if (rc != SAE_OK) return rc;
    }
    ema_advance_kernel<<<1, 1, 0, st>>>(updates, skip);
    return check_launch("ema_advance");
}
