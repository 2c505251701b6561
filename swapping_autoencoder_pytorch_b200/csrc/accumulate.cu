// Gradient accumulation into the flat bucket (SwappingAutoencoderOptimizer with opt.micro_batches > 1): one update sums the
// gradients of several micro-batches.  Micro-batch 0 is copied into the bucket by sae_bucket_pack; every later one is added by
// sae_bucket_accumulate, in the same layout, and Adam reads the bucket views (grad_scale = 1 / (micro_batches * world)).
#include "common.cuh"

namespace sae {

constexpr int ACC_THREADS = 256;
// enough blocks that the largest tensor alone (a third of the generator's group) keeps every SM streaming; the blocks of a small
// tensor that find no element exit at once
constexpr int ACC_BLOCKS_PER_TENSOR = 256;

__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

// One grid row (blockIdx.y) per tensor, grid-stride over its elements: bucket[offsets[t] + i] += ptrs[t][i].  When the gradient
// and its bucket segment are both 16-byte aligned (segments always are; a gradient view may not be) the first 4 * (size / 4)
// elements go as float4, the gradient read with a streaming load (it is not read again); the rest, and every element of an
// unaligned tensor, one by one.  Each element is one round-to-nearest fp32 add, so the result is bitwise torch's a + b and does
// not depend on the schedule: no atomics, no shared memory, and deterministic mode needs no twin.
__global__ void __launch_bounds__(ACC_THREADS)
bucket_accumulate_kernel(const float* const* __restrict__ ptrs, const int64_t* __restrict__ offsets,
                         const int64_t* __restrict__ sizes, float* __restrict__ bucket) {
    const int t = blockIdx.y;
    const float* g = ptrs[t];
    if (g == nullptr) return;
    float* b = bucket + offsets[t];
    const int64_t size = sizes[t];
    const int64_t first = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    int64_t tail = 0;
    if (((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(b)) & 15) == 0) {
        const int64_t n4 = size / 4;
        const float4* g4 = reinterpret_cast<const float4*>(g);
        float4* b4 = reinterpret_cast<float4*>(b);
        int64_t i = first;
        for (; i + stride < n4; i += 2 * stride) {           // two independent float4 pairs in flight per thread
            const float4 v0 = ldg_stream(g4 + i), v1 = ldg_stream(g4 + i + stride);
            const float4 a0 = b4[i], a1 = b4[i + stride];
            b4[i] = add4(a0, v0);
            b4[i + stride] = add4(a1, v1);
        }
        if (i < n4) b4[i] = add4(b4[i], ldg_stream(g4 + i));
        tail = n4 * 4;
    }
    for (int64_t i = tail + first; i < size; i += stride) b[i] = __fadd_rn(b[i], __ldg(g + i));
}

}  // namespace sae

using namespace sae;

extern "C" int sae_bucket_accumulate(const float* const* ptrs, const int64_t* offsets, const int64_t* sizes, int n,
                                     float* bucket, int64_t total, void* stream) {
    if (n == 0) return SAE_OK;
    if (!ptrs || !offsets || !sizes || !bucket || n < 0 || total < 0)
        return fail(SAE_E_INVALID, "bucket_accumulate: bad arguments");
    if (n > 65535) return fail(SAE_E_UNSUPPORTED, "bucket_accumulate: more than 65535 tensors in one table");
    dim3 grid(ACC_BLOCKS_PER_TENSOR, (unsigned)n);
    bucket_accumulate_kernel<<<grid, ACC_THREADS, 0, (cudaStream_t)stream>>>(ptrs, offsets, sizes, bucket);
    return check_launch("bucket_accumulate");
}
