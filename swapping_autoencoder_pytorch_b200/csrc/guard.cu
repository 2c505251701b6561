// Non-finite scan of the gradients a half-step is about to hand to Adam (the skip-on-non-finite guard,
// SwappingAutoencoderOptimizer with opt.skip_nonfinite_steps): counts the NaN / +Inf / -Inf elements of every tensor of a
// pointer table, per tensor and in total.  sae_adam_step_guarded reads the total on the device and drops the update when it
// is non-zero, so the decision never reaches the host.
#include "common.cuh"

namespace sae {

// exponent field all ones: +-Inf or NaN.  +-FLT_MAX, denormals and -0.0 are finite.
__device__ __forceinline__ unsigned nonfinite(float v) {
    return (__float_as_uint(v) & 0x7f800000u) == 0x7f800000u;
}

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_BLOCKS_PER_TENSOR = 48;

// One grid row (blockIdx.y) per tensor, grid-stride over its elements.  A 16-byte aligned tensor is read as float4 over its
// first 4 * (size / 4) elements, the last size % 4 elements one by one; an unaligned one is read element by element.  Each block
// sums its threads' counts with warp shuffles and plain shared-memory stores, and only a block that found something touches
// global memory: one integer atomic into the tensor's entry, one into the total.  Integer sums are exact in any order, so the
// result does not depend on the schedule.
__global__ void __launch_bounds__(SCAN_THREADS)
nonfinite_count_kernel(const float* const* __restrict__ ptrs, const int64_t* __restrict__ sizes, int n,
                       unsigned long long* __restrict__ counts) {
    const int t = blockIdx.y;
    const float* x = ptrs[t];
    if (x == nullptr) return;
    const int64_t size = sizes[t];
    const int64_t first = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    unsigned long long c = 0;
    int64_t tail = 0;
    if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
        const int64_t n4 = size / 4;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        for (int64_t i = first; i < n4; i += stride) {
            const float4 v = ldg_stream(x4 + i);
            c += nonfinite(v.x) + nonfinite(v.y) + nonfinite(v.z) + nonfinite(v.w);
        }
        tail = n4 * 4;
    }
    for (int64_t i = tail + first; i < size; i += stride) c += nonfinite(__ldg(x + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    __shared__ unsigned long long warp_count[SCAN_THREADS / 32];
    if ((threadIdx.x & 31) == 0) warp_count[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long s = 0;
#pragma unroll
        for (int w = 0; w < SCAN_THREADS / 32; ++w) s += warp_count[w];
        if (s) {
            atomicAdd(counts + t, s);
            atomicAdd(counts + n, s);
        }
    }
}

}  // namespace sae

using namespace sae;

extern "C" int sae_nonfinite_count(const float* const* ptrs, const int64_t* sizes, int n, unsigned long long* counts,
                                   void* stream) {
    if (n == 0) return SAE_OK;
    if (!ptrs || !sizes || !counts || n < 0) return fail(SAE_E_INVALID, "nonfinite_count: bad arguments");
    if (n > 65535) return fail(SAE_E_UNSUPPORTED, "nonfinite_count: more than 65535 tensors in one table");
    dim3 grid(SCAN_BLOCKS_PER_TENSOR, (unsigned)n);
    nonfinite_count_kernel<<<grid, SCAN_THREADS, 0, (cudaStream_t)stream>>>(ptrs, sizes, n, counts);
    return check_launch("nonfinite_count");
}
