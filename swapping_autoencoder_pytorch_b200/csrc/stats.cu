// Training statistics (SwappingAutoencoderOptimizer with opt.training_stats; INTEGRATION §2g): device-side fp64 sums that a
// window accumulates across half-steps and the host reads once, when the user asks.
//   * sae_sumsq: per-tensor sum of squares over a pointer table (the gradients Adam reads, grad_scale folded in);
//   * sae_adam_norms: per-tensor sums of squares of the parameters and of the step Adam just applied to them, the step
//     recomputed from the moments and step counts with the Adam kernel's own fp32 expression (train_ops.cu);
//   * sae_score_stats: sum, sum of signs, finite and non-finite counts of one discriminator logit tensor.
// None of them uses a float atomic: a tensor's elements are split over SAE_STATS_BLOCKS blocks by a partition that depends on
// its size alone, every block stores its partial into a caller-provided workspace, and a second launch adds each tensor's
// partials in block order.  The results are therefore bitwise reproducible, and deterministic mode needs no twin.
#include <cmath>

#include "common.cuh"

namespace sae {

constexpr int STATS_THREADS = 256;
constexpr int STATS_BLOCKS = SAE_STATS_BLOCKS;
static_assert(STATS_BLOCKS % 32 == 0, "the finishing warp reads the partials 32 at a time");

// sum of the block's per-thread values in a fixed order (xor butterfly inside each warp, then the warps in index order);
// the result is valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __shared__ double warp_part[STATS_THREADS / 32];
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 0; w < STATS_THREADS / 32; ++w) s += warp_part[w];
    }
    __syncthreads();            // warp_part is reused by the next call
    return s;
}

// Elements 4j .. 4j+3 of a tensor of `size` elements, for j < size / 4, go to thread j mod (STATS_BLOCKS * STATS_THREADS) of
// the tensor's grid row, in increasing j; the last size % 4 elements to threads 0, 1, 2.  The group is read as one float4 when
// the address is 16-byte aligned and as four scalars otherwise, and its four squares are added in element order either way:
// the partition and the order of every addition depend on the size alone, not on the alignment of the view.
__device__ __forceinline__ float4 load4(const float* x, int64_t j, bool aligned) {
    if (aligned) return ldg_stream(reinterpret_cast<const float4*>(x) + j);
    return make_float4(__ldg(x + 4 * j), __ldg(x + 4 * j + 1), __ldg(x + 4 * j + 2), __ldg(x + 4 * j + 3));
}

__device__ __forceinline__ double sq4(double acc, float4 v) {
    acc = fma((double)v.x, (double)v.x, acc);
    acc = fma((double)v.y, (double)v.y, acc);
    acc = fma((double)v.z, (double)v.z, acc);
    return fma((double)v.w, (double)v.w, acc);
}

// partials[t * STATS_BLOCKS + blockIdx.x] = the block's sum of x_t[i]^2 (0 for a block past the end of the tensor)
__global__ void __launch_bounds__(STATS_THREADS)
sumsq_kernel(const float* const* __restrict__ ptrs, const int64_t* __restrict__ sizes, double* __restrict__ partials,
             const unsigned long long* __restrict__ skip) {
    if (skip && *skip) return;
    const int t = blockIdx.y;
    const float* x = ptrs[t];
    if (x == nullptr) return;
    const int64_t size = sizes[t], n4 = size / 4;
    const int64_t first = blockIdx.x * (int64_t)STATS_THREADS + threadIdx.x, stride = (int64_t)STATS_BLOCKS * STATS_THREADS;
    const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    double acc = 0.0;
    int64_t j = first;
    for (; j + stride < n4; j += 2 * stride) {            // two independent loads in flight per thread
        const float4 a = load4(x, j, aligned), b = load4(x, j + stride, aligned);
        acc = sq4(sq4(acc, a), b);
    }
    if (j < n4) acc = sq4(acc, load4(x, j, aligned));
    if (first < size - 4 * n4) {
        const float v = __ldg(x + 4 * n4 + first);
        acc = fma((double)v, (double)v, acc);
    }
    const double s = block_sum(acc);
    if (threadIdx.x == 0) partials[(int64_t)t * STATS_BLOCKS + blockIdx.x] = s;
}

// Sum of `rows` rows of STATS_BLOCKS partials, one warp per row in a fixed order; out[row] += scale2 * sum.  Rows whose
// tensor pointer is NULL are left alone (their partials were never written).  One thread also advances *updates.
__global__ void __launch_bounds__(STATS_THREADS)
stats_finish_kernel(const double* __restrict__ partials, int rows, const float* const* __restrict__ ptrs, int rows_per_ptr,
                    double* out0, double* out1, double scale2, double* __restrict__ updates,
                    const unsigned long long* __restrict__ skip) {
    if (skip && *skip) return;
    if (updates && blockIdx.x == 0 && threadIdx.x == 0) *updates += 1.0;
    const int row = blockIdx.x * (STATS_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int t = row / rows_per_ptr;
    if (ptrs[t] == nullptr) return;
    const double* p = partials + (int64_t)row * STATS_BLOCKS;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < STATS_BLOCKS / 32; ++k) s += p[k * 32 + lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
        double* out = (row % rows_per_ptr == 0) ? out0 : out1;
        out[t] += scale2 * s;
    }
}

// Squares of the parameter and of Adam's step after an update, in the partition of sumsq_kernel.  The step is the Adam
// kernel's expression on the stored (updated) moments and the advanced step count:  step_size * m / (sqrtf(v) / bc2_sqrt +
// eps).  partials row 2t: the parameter; row 2t + 1: the step (0 for a tensor without gradient, which Adam skipped).
__device__ __forceinline__ float adam_delta(float m, float v, float step_size, float bc2_sqrt, float eps) {
    return step_size * m / (sqrtf(v) / bc2_sqrt + eps);
}

__global__ void __launch_bounds__(STATS_THREADS)
adam_norms_kernel(const float* const* __restrict__ p_ptrs, const float* const* __restrict__ g_ptrs,
                  const int64_t* __restrict__ offsets, const int64_t* __restrict__ sizes, const float* __restrict__ exp_avg,
                  const float* __restrict__ exp_avg_sq, const float* __restrict__ steps, float lr, float b1, float b2, float eps,
                  double* __restrict__ partials, const unsigned long long* __restrict__ skip) {
    if (skip && *skip) return;
    const int t = blockIdx.y;
    const float* p = p_ptrs[t];
    if (p == nullptr) return;
    const bool stepped = g_ptrs[t] != nullptr;
    const float* m = exp_avg + offsets[t];
    const float* v = exp_avg_sq + offsets[t];
    const int64_t size = sizes[t], n4 = size / 4;
    const int64_t first = blockIdx.x * (int64_t)STATS_THREADS + threadIdx.x, stride = (int64_t)STATS_BLOCKS * STATS_THREADS;
    const bool p_aligned = (reinterpret_cast<uintptr_t>(p) & 15) == 0;
    const bool mv_aligned = ((reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    // the step count after the update equals the Adam kernel's  steps[t] + 1.f  before it
    const float step = steps[t];
    const float bc1 = 1.f - powf(b1, step);
    const float bc2_sqrt = sqrtf(1.f - powf(b2, step));
    const float step_size = lr / bc1;
    double wacc = 0.0, uacc = 0.0;
    for (int64_t j = first; j < n4; j += stride) {
        wacc = sq4(wacc, load4(p, j, p_aligned));
        if (stepped) {
            const float4 mm = load4(m, j, mv_aligned), vv = load4(v, j, mv_aligned);
            uacc = sq4(uacc, make_float4(adam_delta(mm.x, vv.x, step_size, bc2_sqrt, eps),
                                         adam_delta(mm.y, vv.y, step_size, bc2_sqrt, eps),
                                         adam_delta(mm.z, vv.z, step_size, bc2_sqrt, eps),
                                         adam_delta(mm.w, vv.w, step_size, bc2_sqrt, eps)));
        }
    }
    if (first < size - 4 * n4) {
        const int64_t i = 4 * n4 + first;
        const float w = __ldg(p + i);
        wacc = fma((double)w, (double)w, wacc);
        if (stepped) {
            const float d = adam_delta(__ldg(m + i), __ldg(v + i), step_size, bc2_sqrt, eps);
            uacc = fma((double)d, (double)d, uacc);
        }
    }
    const double ws = block_sum(wacc), us = block_sum(uacc);
    if (threadIdx.x == 0) {
        partials[(2 * (int64_t)t) * STATS_BLOCKS + blockIdx.x] = ws;
        partials[(2 * (int64_t)t + 1) * STATS_BLOCKS + blockIdx.x] = us;
    }
}

// ---------------------------------------------------------------------------------------------------- score statistics
struct ScoreView {
    const float* x;
    int64_t size[4], stride[4];      // outermost first; unused dimensions have size 1
    int64_t numel;
};

// One block.  Element e (row-major over the logical shape) goes to thread e mod STATS_THREADS, in increasing e; the block then
// sums in a fixed order and thread 0 adds into acc.  Non-finite elements are counted and left out of both sums.
__global__ void __launch_bounds__(STATS_THREADS)
score_stats_kernel(const ScoreView s, double* __restrict__ acc) {
    double sum = 0.0, sgn = 0.0, fin = 0.0, bad = 0.0;
    for (int64_t e = threadIdx.x; e < s.numel; e += STATS_THREADS) {
        int64_t r = e, off = 0;
#pragma unroll
        for (int d = 3; d >= 0; --d) {
            off += (r % s.size[d]) * s.stride[d];
            r /= s.size[d];
        }
        const float v = __ldg(s.x + off);
        if ((__float_as_uint(v) & 0x7f800000u) == 0x7f800000u) {
            bad += 1.0;
        } else {
            sum += (double)v;
            sgn += (v > 0.f) ? 1.0 : ((v < 0.f) ? -1.0 : 0.0);
            fin += 1.0;
        }
    }
    sum = block_sum(sum);
    sgn = block_sum(sgn);
    fin = block_sum(fin);
    bad = block_sum(bad);
    if (threadIdx.x == 0) {
        acc[0] += sum;
        acc[1] += sgn;
        acc[2] += fin;
        acc[3] += bad;
    }
}

}  // namespace sae

using namespace sae;

static int stats_table_args(int n, const char* who) {
    if (n < 0 || n > 65535) return fail(SAE_E_INVALID, "%s: n = %d outside [0, 65535]", who, n);
    return SAE_OK;
}

extern "C" int sae_sumsq(const float* const* ptrs, const int64_t* sizes, int n, float scale, double* out, double* partials,
                         const unsigned long long* skip, void* stream) {
    int rc = stats_table_args(n, "sumsq");
    if (rc) return rc;
    if (!ptrs || !sizes || !out || !partials) return fail(SAE_E_INVALID, "sumsq: null pointer");
    if (!std::isfinite(scale)) return fail(SAE_E_INVALID, "sumsq: scale must be finite");
    if (n == 0) return SAE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    sumsq_kernel<<<dim3(STATS_BLOCKS, (unsigned)n), STATS_THREADS, 0, st>>>(ptrs, sizes, partials, skip);
    rc = check_launch("sumsq");
    if (rc) return rc;
    const double s = (double)scale;
    stats_finish_kernel<<<(n + STATS_THREADS / 32 - 1) / (STATS_THREADS / 32), STATS_THREADS, 0, st>>>(
        partials, n, ptrs, 1, out, out, s * s, nullptr, skip);
    return check_launch("sumsq_finish");
}

extern "C" int sae_adam_norms(const float* const* p_ptrs, const float* const* g_ptrs, const int64_t* offsets,
                              const int64_t* sizes, int n, const float* exp_avg, const float* exp_avg_sq, const float* steps,
                              float lr, float beta1, float beta2, float eps, double* weight_out, double* update_out,
                              double* updates, double* partials, const unsigned long long* skip, void* stream) {
    int rc = stats_table_args(n, "adam_norms");
    if (rc) return rc;
    if (!p_ptrs || !g_ptrs || !offsets || !sizes || !exp_avg || !exp_avg_sq || !steps || !weight_out || !update_out || !partials)
        return fail(SAE_E_INVALID, "adam_norms: null pointer");
    if (!(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f))
        return fail(SAE_E_INVALID, "adam_norms: betas must lie in [0, 1) and eps must be >= 0");
    cudaStream_t st = (cudaStream_t)stream;
    if (n > 0) {
        adam_norms_kernel<<<dim3(STATS_BLOCKS, (unsigned)n), STATS_THREADS, 0, st>>>(
            p_ptrs, g_ptrs, offsets, sizes, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, partials, skip);
        rc = check_launch("adam_norms");
        if (rc) return rc;
    }
    if (n == 0 && !updates) return SAE_OK;
    const int rows = 2 * n;
    stats_finish_kernel<<<rows > 0 ? (rows + STATS_THREADS / 32 - 1) / (STATS_THREADS / 32) : 1, STATS_THREADS, 0, st>>>(
        partials, rows, p_ptrs, 2, weight_out, update_out, 1.0, updates, skip);
    return check_launch("adam_norms_finish");
}

extern "C" int sae_score_stats(const float* x, int ndim, const int64_t* sizes, const int64_t* strides, double* acc,
                               void* stream) {
    if (!acc || !sizes || !strides || ndim < 1 || ndim > 4) return fail(SAE_E_INVALID, "score_stats: bad arguments");
    ScoreView s;
    s.x = x;
    s.numel = 1;
    for (int d = 0; d < 4; ++d) {
        const int k = d - (4 - ndim);            // the given dimensions fill the innermost slots
        s.size[d] = k >= 0 ? sizes[k] : 1;
        s.stride[d] = k >= 0 ? strides[k] : 0;
        if (s.size[d] < 0 || s.stride[d] < 0) return fail(SAE_E_INVALID, "score_stats: negative size or stride");
        s.numel *= s.size[d];
    }
    if (s.numel == 0) return SAE_OK;
    if (!x) return fail(SAE_E_INVALID, "score_stats: null pointer");
    score_stats_kernel<<<1, STATS_THREADS, 0, (cudaStream_t)stream>>>(s, acc);
    return check_launch("score_stats");
}
