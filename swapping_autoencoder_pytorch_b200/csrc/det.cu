// Deterministic twins of the bandwidth-bound backward passes that reduce across CTAs (sae_bias_act_backward,
// sae_modulate_backward, sae_fir_act_backward, sae_torgb_backward): see "Deterministic mode" in include/sae_b200.h.
//
// The atomic kernels (elementwise.cu, torgb.cu, upfirdn2d.cu) sum inside a CTA with shared-memory atomics and across CTAs
// with fp32 global atomics.  Here nothing is atomic:
//   * inside a CTA, every thread's partial sums go to a shared-memory row [thread][VEC] and one thread per channel adds the
//     rows of the threads that own that channel in thread order (warp order, then lane order);
//   * across CTAs, each CTA stores its sums with plain stores into its workspace slot, ws[slot][target], and det_reduce adds
//     the slots into the destination in slot order.
// Grids are planned for DET_SMS SMs, so the partition, and with it the order of every addition, is a function of the
// arguments alone.  The loops over the data are those of the atomic kernels, so grad_in / dx of the bias / activation,
// modulation and ToRGB twins are bitwise equal to theirs.
#include "common.cuh"

namespace sae {

static unsigned det_blocks(int64_t work, int per_sm) {
    int64_t b = (work + 255) / 256;
    if (b > (int64_t)DET_SMS * per_sm) b = (int64_t)DET_SMS * per_sm;
    return (unsigned)(b < 1 ? 1 : b);
}

// ---------------------------------------------------------------------------- bias_act backward
// grad_in = grad_out * (out > 0 ? 1 : alpha) * scale (or the branch from act_mask); slot blockIdx.x of ws_gb ([C] floats) gets
// this CTA's per-channel sums, slot blockIdx.x of ws_nw (1 float) its noise-weight sum.  grad_in may alias grad_out.
template <int VEC>
__global__ void __launch_bounds__(256)
bias_act_bwd_det_kernel(const float* go, const float* __restrict__ outp, float* gi, float* __restrict__ ws_gb, int64_t size_v,
                        int cv, int64_t stride_v, float alpha, float scale, const float* __restrict__ noise, int64_t noise_div,
                        float* __restrict__ ws_nw, int round_tf32, const uint32_t* __restrict__ act_mask) {
    __shared__ float rows[256 * VEC];
    __shared__ float wsum[8];
    const int C = cv * VEC;
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    float bsum[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) bsum[j] = 0.f;
    float nsum = 0.f;
    if (tid < stride_v) {
        for (int64_t i = tid; i < size_v; i += stride_v) {
            float g[VEC], o[VEC];
            if (VEC == 4) {
                float4 t = reinterpret_cast<const float4*>(go)[i];
                g[0] = t.x; g[1 % VEC] = t.y; g[2 % VEC] = t.z; g[3 % VEC] = t.w;
                if (act_mask) {
                    const uint32_t wd = __ldg(act_mask + (i >> 3)) >> (((uint32_t)i & 7u) * 4u);
                    o[0] = (wd & 1u) ? 1.f : 0.f; o[1 % VEC] = (wd & 2u) ? 1.f : 0.f; o[2 % VEC] = (wd & 4u) ? 1.f : 0.f; o[3 % VEC] = (wd & 8u) ? 1.f : 0.f;
                } else {
                    float4 q = ldg_stream(reinterpret_cast<const float4*>(outp) + i);
                    o[0] = q.x; o[1 % VEC] = q.y; o[2 % VEC] = q.z; o[3 % VEC] = q.w;
                }
            } else {
                g[0] = go[i]; o[0] = outp[i];
            }
            float lsum = 0.f;
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
                float y = ((o[j] > 0.f) ? g[j] : g[j] * alpha) * scale;
                g[j] = round_tf32 ? rna_tf32(y) : y;
                bsum[j] += y;
                lsum += y;
            }
            if (noise) nsum = fmaf(lsum, __ldg(noise + (i * VEC) / noise_div), nsum);
            if (VEC == 4) reinterpret_cast<float4*>(gi)[i] = make_float4(g[0], g[1 % VEC], g[2 % VEC], g[3 % VEC]);
            else gi[i] = g[0];
        }
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) rows[threadIdx.x * VEC + j] = bsum[j];      // zero for threads past stride_v
    if (noise) {
        nsum = warp_sum(nsum);
        if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = nsum;
    }
    __syncthreads();
    if (ws_gb) {
        // channel group q is served by the threads t = t0 + k cv of this CTA (global thread index = q mod cv)
        const int base = (int)(((int64_t)blockIdx.x * blockDim.x) % cv);
        for (int i = threadIdx.x; i < C; i += blockDim.x) {
            const int q = i / VEC, j = i - q * VEC;
            float v = 0.f;
            for (int t = (q - base + cv) % cv; t < (int)blockDim.x; t += cv) v += rows[t * VEC + j];
            ws_gb[(int64_t)blockIdx.x * C + i] = v;
        }
    }
    if (noise && threadIdx.x == 0) {
        float v = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += wsum[w];
        ws_nw[blockIdx.x] = v;
    }
}

// --------------------------------------------------------------------------------- modulate backward
// dx = dy * s; slot blockIdx.x (pixel chunk) of ws ([N, C] floats) gets sum_{chunk pixels} dy * x of sample blockIdx.y.
// Narrow rows (cv <= 256): threads own a fixed channel group, shared rows added in thread order.  Wide rows: every thread
// owns whole channel groups and walks the chunk's pixels in order.
template <int VEC>
__global__ void __launch_bounds__(256)
modulate_bwd_det_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ s,
                        float* __restrict__ dx, float* __restrict__ ws, int64_t hw, int cv, int64_t pix_per_cta, int round_tf32) {
    __shared__ float rows[256 * VEC];
    const int C = cv * VEC;
    const int n = blockIdx.y;
    const int64_t p0 = blockIdx.x * pix_per_cta;
    int64_t p1 = p0 + pix_per_cta;
    if (p1 > hw) p1 = hw;
    const int64_t base_v = (int64_t)n * hw * cv;
    const int64_t lo = p0 * cv, hi = p1 * cv;
    float* slot = ws + ((int64_t)blockIdx.x * gridDim.y + n) * C;
    const int stride = (int)(blockDim.x / cv) * cv;
    if (stride > 0) {
        float acc[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
        if ((int)threadIdx.x < stride) {
            const int c = threadIdx.x % cv;
            float m[VEC];
#pragma unroll
            for (int j = 0; j < VEC; ++j) m[j] = __ldg(s + (int64_t)n * C + c * VEC + j);
            for (int64_t i = lo + threadIdx.x; i < hi; i += stride) {
                float g[VEC], a[VEC];
                if (VEC == 4) {
                    float4 t = ldg_stream(reinterpret_cast<const float4*>(dy) + base_v + i);
                    float4 q = ldg_stream(reinterpret_cast<const float4*>(x) + base_v + i);
                    g[0] = t.x; g[1 % VEC] = t.y; g[2 % VEC] = t.z; g[3 % VEC] = t.w;
                    a[0] = q.x; a[1 % VEC] = q.y; a[2 % VEC] = q.z; a[3 % VEC] = q.w;
                } else {
                    g[0] = dy[base_v + i]; a[0] = x[base_v + i];
                }
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                    acc[j] = fmaf(g[j], a[j], acc[j]);
                    g[j] = round_tf32 ? rna_tf32(g[j] * m[j]) : g[j] * m[j];
                }
                if (VEC == 4) reinterpret_cast<float4*>(dx)[base_v + i] = make_float4(g[0], g[1 % VEC], g[2 % VEC], g[3 % VEC]);
                else dx[base_v + i] = g[0];
            }
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) rows[threadIdx.x * VEC + j] = acc[j];
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) {
            const int q = i / VEC, j = i - q * VEC;
            float v = 0.f;
            for (int t = q; t < stride; t += cv) v += rows[t * VEC + j];
            slot[i] = v;
        }
        return;
    }
    for (int q = threadIdx.x; q < cv; q += blockDim.x) {
        float m[VEC], a[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) { m[j] = __ldg(s + (int64_t)n * C + q * VEC + j); a[j] = 0.f; }
        for (int64_t i = lo + q; i < hi; i += cv) {
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
                const int64_t e = (base_v + i) * VEC + j;
                const float g = dy[e];
                a[j] = fmaf(g, x[e], a[j]);
                const float d = g * m[j];
                dx[e] = round_tf32 ? rna_tf32(d) : d;
            }
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) slot[q * VEC + j] = a[j];
    }
}

// ---------------------------------------------------------------------------------------- ToRGB backward
// the loop of torgb_bwd_kernel; slot = the strip index inside the sample, [N, 3, C] floats per slot, written by the warp that
// owns strip (n, slot)
constexpr int TORGB_DET_MAXJ = 8;

template <int NJ>
__global__ void __launch_bounds__(256)
torgb_bwd_det_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ s, const float* __restrict__ w,
                     float* __restrict__ dx, float* __restrict__ ws, int N, int64_t HW, int W_img, int C, int strips_per_sample,
                     float wscale, int64_t ds_n, int64_t ds_c, int64_t ds_h, int64_t ds_w, int round_tf32) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t warps_total = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t strip_len = (HW + strips_per_sample - 1) / strips_per_sample;
    for (int64_t item = warp_global; item < (int64_t)N * strips_per_sample; item += warps_total) {
        const int n = (int)(item / strips_per_sample);
        const int64_t p_begin = (item % strips_per_sample) * strip_len;
        const int64_t p_end = min(p_begin + strip_len, HW);
        float wc[NJ][3][4], g[NJ][3][4];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int c = 4 * lane + 128 * j;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float sv = (c + u < C) ? __ldg(s + (int64_t)n * C + c + u) * wscale : 0.f;
#pragma unroll
                for (int o = 0; o < 3; ++o) {
                    wc[j][o][u] = (c + u < C) ? sv * __ldg(w + (int64_t)o * C + c + u) : 0.f;
                    g[j][o][u] = 0.f;
                }
            }
        }
        const float* xn = x + (int64_t)n * HW * C;
        float* dxn = dx ? dx + (int64_t)n * HW * C : nullptr;
        const float* dyn = dy + (int64_t)n * ds_n;
        for (int64_t p = p_begin; p < p_end; ++p) {
            const int64_t ph = p / W_img, pw = p - ph * W_img;
            const float* d = dyn + ph * ds_h + pw * ds_w;
            const float d0 = __ldg(d), d1 = __ldg(d + ds_c), d2 = __ldg(d + 2 * ds_c);
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int c = 4 * lane + 128 * j;
                if (c < C) {
                    if (ws) {
                        const float4 v = ldg_stream(reinterpret_cast<const float4*>(xn + p * C + c));
                        g[j][0][0] += d0 * v.x; g[j][0][1] += d0 * v.y; g[j][0][2] += d0 * v.z; g[j][0][3] += d0 * v.w;
                        g[j][1][0] += d1 * v.x; g[j][1][1] += d1 * v.y; g[j][1][2] += d1 * v.z; g[j][1][3] += d1 * v.w;
                        g[j][2][0] += d2 * v.x; g[j][2][1] += d2 * v.y; g[j][2][2] += d2 * v.z; g[j][2][3] += d2 * v.w;
                    }
                    if (dxn) {
                        float4 o;
                        o.x = d0 * wc[j][0][0] + d1 * wc[j][1][0] + d2 * wc[j][2][0];
                        o.y = d0 * wc[j][0][1] + d1 * wc[j][1][1] + d2 * wc[j][2][1];
                        o.z = d0 * wc[j][0][2] + d1 * wc[j][1][2] + d2 * wc[j][2][2];
                        o.w = d0 * wc[j][0][3] + d1 * wc[j][1][3] + d2 * wc[j][2][3];
                        if (round_tf32) { o.x = rna_tf32(o.x); o.y = rna_tf32(o.y); o.z = rna_tf32(o.z); o.w = rna_tf32(o.w); }
                        *reinterpret_cast<float4*>(dxn + p * C + c) = o;
                    }
                }
            }
        }
        if (ws) {
            float* const gn = ws + ((item - (int64_t)n * strips_per_sample) * N + n) * 3 * C;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int c = 4 * lane + 128 * j;
#pragma unroll
                for (int o = 0; o < 3; ++o)
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        if (c + u < C) gn[o * C + c + u] = g[j][o][u];
            }
        }
    }
}

}  // namespace sae

using namespace sae;

extern "C" int sae_bias_act_backward_det(const float* grad_out, const float* out, float* grad_in, float* grad_bias,
                                         int64_t size_x, int size_b, float alpha, float scale,
                                         const float* noise, int64_t noise_div, float* grad_noise_weight,
                                         int round_tf32, const uint32_t* act_mask, void* workspace, int64_t* workspace_bytes,
                                         void* stream) {
    const char* who = "bias_act_backward_det";
    bool query;
    if (size_x == 0) return det_workspace(workspace, workspace_bytes, 0, who, &query);
    if (!grad_out || (!out && !act_mask) || !grad_in || size_b <= 0 || size_x % size_b != 0)
        return fail(SAE_E_INVALID, "%s: bad arguments (size_x %% size_b must be 0)", who);
    if (act_mask && size_b % 32 != 0) return fail(SAE_E_INVALID, "%s: the activation bit mask needs a channel count that is a multiple of 32", who);
    if (noise && (!grad_noise_weight || noise_div <= 0)) return fail(SAE_E_INVALID, "%s: noise needs grad slot", who);
    if (size_b > 12000) return fail(SAE_E_UNSUPPORTED, "%s: more than 12000 channels", who);
    uintptr_t al = reinterpret_cast<uintptr_t>(grad_out) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(grad_in);
    const bool vec = (size_b % 4 == 0) && (al % 16 == 0) && (!noise || noise_div % 4 == 0);
    if (act_mask && !vec) return fail(SAE_E_INVALID, "%s: the activation bit mask needs the vectorised path (16-byte aligned pointers)", who);
    const int V = vec ? 4 : 1;
    const int cv = size_b / V;
    const int64_t size_v = size_x / V;
    unsigned blocks = det_blocks(size_v, 4);
    int64_t threads = (int64_t)blocks * 256;
    int64_t stride = (threads / cv) * cv;       // a multiple of cv: each thread's channel group is loop-invariant
    if (stride == 0) {
        blocks = (unsigned)((cv + 255) / 256);
        threads = (int64_t)blocks * 256;
        stride = (threads / cv) * cv;
    }
    // workspace: grad_bias slots [blocks][size_b], then grad_noise_weight slots [blocks]
    const int64_t gb_bytes = grad_bias ? det_region((int64_t)blocks * size_b) : 0;
    int rc = det_workspace(workspace, workspace_bytes, gb_bytes + (noise ? det_region(blocks) : 0), who, &query);
    if (rc || query) return rc;
    float* ws_gb = grad_bias ? static_cast<float*>(workspace) : nullptr;
    float* ws_nw = reinterpret_cast<float*>(static_cast<char*>(workspace) + gb_bytes);
    cudaStream_t st = (cudaStream_t)stream;
    if (vec)
        bias_act_bwd_det_kernel<4><<<blocks, 256, 0, st>>>(grad_out, out, grad_in, ws_gb, size_v, cv, stride, alpha, scale, noise,
                                                          noise_div, ws_nw, round_tf32, act_mask);
    else
        bias_act_bwd_det_kernel<1><<<blocks, 256, 0, st>>>(grad_out, out, grad_in, ws_gb, size_v, cv, stride, alpha, scale, noise,
                                                          noise_div, ws_nw, round_tf32, nullptr);
    rc = check_launch(who);
    if (rc == SAE_OK && grad_bias) rc = det_reduce(grad_bias, ws_gb, blocks, size_b, true, 0, st);
    if (rc == SAE_OK && noise) rc = det_reduce(grad_noise_weight, ws_nw, blocks, 1, true, 0, st);
    return rc;
}

extern "C" int sae_modulate_backward_det(const float* dy, const float* x, const float* s, float* dx, float* ds,
                                         int n, int64_t hw, int c, int round_tf32, void* workspace, int64_t* workspace_bytes,
                                         void* stream) {
    const char* who = "modulate_backward_det";
    bool query;
    if (n == 0 || hw == 0) return det_workspace(workspace, workspace_bytes, 0, who, &query);
    if (!dy || !x || !s || !dx || !ds || n < 0 || c <= 0) return fail(SAE_E_INVALID, "%s: bad arguments", who);
    if (c > 12000) return fail(SAE_E_UNSUPPORTED, "%s: more than 12000 channels", who);
    uintptr_t al = reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dx);
    const bool vec = (c % 4 == 0) && (al % 16 == 0);
    const int V = vec ? 4 : 1;
    int64_t want = ((int64_t)DET_SMS * 4 + n - 1) / n;     // ~4 CTAs per SM over the whole batch
    if (want < 1) want = 1;
    int64_t pix_per_cta = (hw + want - 1) / want;
    if (pix_per_cta < 8) pix_per_cta = 8;
    const unsigned chunks = (unsigned)((hw + pix_per_cta - 1) / pix_per_cta);
    // workspace: ds slots [chunks][n][c]
    int rc = det_workspace(workspace, workspace_bytes, det_region((int64_t)chunks * n * c), who, &query);
    if (rc || query) return rc;
    float* w = static_cast<float*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(chunks, (unsigned)n);
    if (vec) modulate_bwd_det_kernel<4><<<grid, 256, 0, st>>>(dy, x, s, dx, w, hw, c / V, pix_per_cta, round_tf32);
    else     modulate_bwd_det_kernel<1><<<grid, 256, 0, st>>>(dy, x, s, dx, w, hw, c / V, pix_per_cta, round_tf32);
    rc = check_launch(who);
    if (rc == SAE_OK) rc = det_reduce(ds, w, chunks, (int64_t)n * c, true, 0, st);
    return rc;
}

// The FIR (sae_upfirdn2d_separable, no reduction, unrounded) into grad_in, then sae_bias_act_backward_det in place on it: one
// more pass over grad_in instead of the fused kernel's atomics.  The negative branch multiplies by alpha, then by scale (the
// fused kernel by alpha * scale), so grad_in may differ from the atomic twin's in the last bit.
extern "C" int sae_fir_act_backward_det(const float* grad, const float* taps_y, const float* taps_x, const float* act_out,
                                        float* grad_in, float* grad_bias, int64_t major, int in_h, int in_w, int minor,
                                        int kernel_h, int kernel_w, int pad_x0, int pad_x1, int pad_y0, int pad_y1,
                                        float alpha, float scale, int round_tf32, const uint32_t* act_mask,
                                        void* workspace, int64_t* workspace_bytes, void* stream) {
    const char* who = "fir_act_backward_det";
    bool query;
    if (major == 0) return det_workspace(workspace, workspace_bytes, 0, who, &query);
    if (!grad || !taps_y || !taps_x || (!act_out && !act_mask) || !grad_in) return fail(SAE_E_INVALID, "%s: null pointer", who);
    if ((kernel_h != 3 && kernel_h != 4) || kernel_w != kernel_h) return fail(SAE_E_UNSUPPORTED, "%s: taps must be 3 or 4, square", who);
    if (minor % 32 != 0 || ((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(grad_in) | reinterpret_cast<uintptr_t>(act_out)) & 15) != 0)
        return fail(SAE_E_UNSUPPORTED, "%s: needs minor %% 32 == 0 and 16-byte aligned pointers", who);
    const int out_h = in_h + pad_y0 + pad_y1 - kernel_h + 1, out_w = in_w + pad_x0 + pad_x1 - kernel_w + 1;
    if (out_h <= 0 || out_w <= 0) return fail(SAE_E_INVALID, "%s: kernel larger than padded input", who);
    const int64_t size_x = major * (int64_t)out_h * out_w * minor;
    int64_t need = 0;
    int rc = sae_bias_act_backward_det(grad_in, act_out, grad_in, grad_bias, size_x, minor, alpha, scale, nullptr, 1, nullptr,
                                       round_tf32, act_mask, nullptr, &need, stream);
    if (rc == SAE_OK) rc = det_workspace(workspace, workspace_bytes, need, who, &query);
    if (rc || query) return rc;
    rc = sae_upfirdn2d_separable(grad, taps_y, taps_x, grad_in, major, in_h, in_w, minor, kernel_h, kernel_w, 1, 1, pad_x0, pad_x1,
                                 pad_y0, pad_y1, 0, stream);
    if (rc) return rc;
    return sae_bias_act_backward_det(grad_in, act_out, grad_in, grad_bias, size_x, minor, alpha, scale, nullptr, 1, nullptr,
                                     round_tf32, act_mask, workspace, workspace_bytes, stream);
}

extern "C" int sae_torgb_backward_det(const float* dy, const float* x, const float* s, const float* w, float* dx, float* gw,
                                      int N, int H, int W, int C, float wscale,
                                      int64_t ds_n, int64_t ds_c, int64_t ds_h, int64_t ds_w, int round_tf32,
                                      void* workspace, int64_t* workspace_bytes, void* stream) {
    const char* who = "torgb_backward_det";
    bool query;
    if (N == 0) return det_workspace(workspace, workspace_bytes, 0, who, &query);
    if (!dy || !x || !s || !w || (!dx && !gw) || N < 0 || H <= 0 || W <= 0) return fail(SAE_E_INVALID, "%s: bad arguments", who);
    if (C <= 0 || C % 4 != 0 || C > 128 * TORGB_DET_MAXJ)
        return fail(SAE_E_UNSUPPORTED, "%s: C must be a multiple of 4, <= %d", who, 128 * TORGB_DET_MAXJ);
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dx)) & 15) return fail(SAE_E_INVALID, "%s: unaligned pointer", who);
    const int64_t HW = (int64_t)H * W;
    // strips as in the atomic twin, planned for DET_SMS SMs: 8 warps x 8 blocks per SM, strips of at least 64 pixels
    int64_t strips = ((int64_t)DET_SMS * 64 + N - 1) / N;
    const int64_t cap_s = HW / 64 > 0 ? HW / 64 : 1;
    if (strips > cap_s) strips = cap_s;
    if (strips < 1) strips = 1;
    int64_t blocks = ((int64_t)N * strips + 7) / 8;
    if (blocks > (int64_t)DET_SMS * 8) blocks = (int64_t)DET_SMS * 8;
    // workspace: gw slots [strips][N, 3, C]
    int rc = det_workspace(workspace, workspace_bytes, gw ? det_region(strips * N * 3 * C) : 0, who, &query);
    if (rc || query) return rc;
    float* ws = gw ? static_cast<float*>(workspace) : nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    const int nj = (C + 127) / 128;
#define SAE_TORGB_BWD_DET(NJ) torgb_bwd_det_kernel<NJ><<<(unsigned)blocks, 256, 0, st>>>(dy, x, s, w, dx, ws, N, HW, W, C, (int)strips, \
                                                                                     wscale, ds_n, ds_c, ds_h, ds_w, round_tf32)
    switch (nj) {
        case 1: SAE_TORGB_BWD_DET(1); break;
        case 2: SAE_TORGB_BWD_DET(2); break;
        case 3: case 4: SAE_TORGB_BWD_DET(4); break;
        default: SAE_TORGB_BWD_DET(8); break;
    }
#undef SAE_TORGB_BWD_DET
    rc = check_launch(who);
    if (rc == SAE_OK && gw) rc = det_reduce(gw, ws, strips, (int64_t)N * 3 * C, true, 0, st);
    return rc;
}
