// Kernels either side of the network passes of a training half-step (SURVEY.md §8 f1 / f2):
//   * multi-tensor Adam over a pointer table (optimizers/swapping_autoencoder_optimizer.py:34-42 builds two torch Adams;
//     here one launch updates a whole parameter group, reading the gradients either from the parameters' own .grad tensors
//     or straight out of the flat all-reduce bucket with the 1/world factor folded in — no unpack pass);
//   * the random-crop resampler of the patch discriminator (util/util.py:323-343: affine grid + F.grid_sample, bilinear,
//     zeros padding, align_corners=False) writing the 32-channel zero-padded NHWC tensor the first Dpatch convolution
//     reads, and its adjoint in gather form (deterministic, no atomics).
#include "common.cuh"

namespace sae {

// ------------------------------------------------------------------------------------------------ Adam
// One grid row (blockIdx.y) per tensor.  torch.optim.Adam semantics (amsgrad off, weight decay 0, maximize off):
//   t <- t + 1;  m <- m + (1 - b1)(g - m);  v <- b2 v + (1 - b2) g^2;
//   p <- p - lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// A tensor whose gradient pointer is null is skipped and keeps its step count, like a parameter whose .grad is None.
// skip (optional, read on the device): when it points at a non-zero count the whole update is dropped — both kernels return
// before touching anything (sae_adam_step_guarded after sae_nonfinite_count).
__global__ void __launch_bounds__(256)
adam_kernel(float* const* __restrict__ p_ptrs, const float* const* __restrict__ g_ptrs, const int64_t* __restrict__ offsets,
            const int64_t* __restrict__ sizes, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
            const float* __restrict__ steps, float lr, float b1, float b2, float eps, float gscale,
            const unsigned long long* __restrict__ skip) {
    if (skip && *skip) return;
    const int t = blockIdx.y;
    const float* g = g_ptrs[t];
    if (g == nullptr) return;
    float* p = p_ptrs[t];
    float* m = exp_avg + offsets[t];
    float* v = exp_avg_sq + offsets[t];
    const int64_t n = sizes[t];
    const float step = steps[t] + 1.f;
    const float bc1 = 1.f - powf(b1, step);
    const float bc2_sqrt = sqrtf(1.f - powf(b2, step));
    const float step_size = lr / bc1;
    const bool vec = (n % 4 == 0) && (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15) == 0);
    if (vec) {
        const int64_t n4 = n / 4;
        float4* p4 = reinterpret_cast<float4*>(p);
        const float4* g4 = reinterpret_cast<const float4*>(g);
        float4* m4 = reinterpret_cast<float4*>(m);
        float4* v4 = reinterpret_cast<float4*>(v);
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            float4 pp = p4[i], gg = g4[i], mm = m4[i], vv = v4[i];
            float* pa = &pp.x; float* ga = &gg.x; float* ma = &mm.x; float* va = &vv.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float gr = ga[j] * gscale;
                ma[j] = ma[j] + (1.f - b1) * (gr - ma[j]);
                va[j] = b2 * va[j] + (1.f - b2) * gr * gr;
                pa[j] -= step_size * ma[j] / (sqrtf(va[j]) / bc2_sqrt + eps);
            }
            p4[i] = pp; m4[i] = mm; v4[i] = vv;
        }
    } else {
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
            const float gr = g[i] * gscale;
            const float mm = m[i] + (1.f - b1) * (gr - m[i]);
            const float vv = b2 * v[i] + (1.f - b2) * gr * gr;
            m[i] = mm; v[i] = vv;
            p[i] -= step_size * mm / (sqrtf(vv) / bc2_sqrt + eps);
        }
    }
}

__global__ void adam_advance_kernel(const float* const* __restrict__ g_ptrs, float* __restrict__ steps, int n,
                                    const unsigned long long* __restrict__ skip) {
    if (skip && *skip) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && g_ptrs[i] != nullptr) steps[i] += 1.f;
}

// ------------------------------------------------------------------------------------------------ crop resampler
// Crop q of the batch (q = image * num_crops + crop) samples image q / num_crops at normalised coordinates
//   gx = (lin_j * flip_q) * sx_q + ox_q,   gy = lin_i * sy_q + oy_q,   lin_k = -1 + 2k / (S - 1)
// and F.grid_sample(align_corners=False) un-normalises them as  ix = ((gx + 1) W - 1) / 2.
struct CropParams {
    const float* flip;      // [Q]
    const float* scale;     // [Q, 2] (x, y)
    const float* offset;    // [Q, 2] (x, y)
    int Q, num_crops, C, H, W, S, CP;
    int64_t xs_n, xs_c, xs_h, xs_w;      // element strides of the source images [B, C, H, W]
    int round_tf32;
};

__device__ __forceinline__ float crop_lin(int k, int S) {
    // torch.linspace(-1, 1, S): start + k * step for the first half, end - (S - 1 - k) * step for the second
    const float step = 2.f / (float)(S - 1);
    return k < S / 2 ? -1.f + step * (float)k : 1.f - step * (float)(S - 1 - k);
}

__global__ void __launch_bounds__(256)
crop_gather_kernel(const float* __restrict__ x, float* __restrict__ out, const CropParams p) {
    // A warp owns 32 consecutive output pixels.  Phase 1: lane l resamples pixel base + l (all lanes busy, 32-bit index
    // arithmetic — the launcher checks the extent).  Phase 2: the warp writes those 32 pixels' 128-byte rows cooperatively,
    // 4 pixels x 8 sixteen-byte slots per store instruction (512 contiguous bytes); slot 0 carries the three channels
    // (fetched from the owning lane with shuffles), slots 1..7 are the zero pad.  CP == 32 here.
    const uint32_t pixels = (uint32_t)p.Q * (uint32_t)p.S * (uint32_t)p.S;
    const uint32_t SS = (uint32_t)p.S * (uint32_t)p.S;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps_total = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t base = warp_global * 32; base < pixels; base += warps_total * 32) {
        const uint32_t idx = base + lane;
        float a[4] = {0.f, 0.f, 0.f, 0.f};
        if (idx < pixels) {
            const uint32_t q = idx / SS, rem = idx - q * SS;
            const int i = (int)(rem / (uint32_t)p.S), j = (int)(rem - (uint32_t)i * (uint32_t)p.S);
            const float gx = (crop_lin(j, p.S) * __ldg(p.flip + q)) * __ldg(p.scale + 2 * q) + __ldg(p.offset + 2 * q);
            const float gy = crop_lin(i, p.S) * __ldg(p.scale + 2 * q + 1) + __ldg(p.offset + 2 * q + 1);
            const float ix = ((gx + 1.f) * (float)p.W - 1.f) * 0.5f;
            const float iy = ((gy + 1.f) * (float)p.H - 1.f) * 0.5f;
            const float fx = floorf(ix), fy = floorf(iy);
            const int x0 = (int)fx, y0 = (int)fy;
            const float tx = ix - fx, ty = iy - fy;
            const float w00 = (1.f - tx) * (1.f - ty), w01 = tx * (1.f - ty), w10 = (1.f - tx) * ty, w11 = tx * ty;
            const bool vx0 = x0 >= 0 && x0 < p.W, vx1 = x0 + 1 >= 0 && x0 + 1 < p.W;
            const bool vy0 = y0 >= 0 && y0 < p.H, vy1 = y0 + 1 >= 0 && y0 + 1 < p.H;
            const float* src = x + (int64_t)(q / (uint32_t)p.num_crops) * p.xs_n;
            const int64_t o00 = (int64_t)y0 * p.xs_h + (int64_t)x0 * p.xs_w;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if (c < p.C) {
                    const float* sc = src + (int64_t)c * p.xs_c + o00;
                    float acc = 0.f;
                    if (vy0 && vx0) acc += w00 * __ldg(sc);
                    if (vy0 && vx1) acc += w01 * __ldg(sc + p.xs_w);
                    if (vy1 && vx0) acc += w10 * __ldg(sc + p.xs_h);
                    if (vy1 && vx1) acc += w11 * __ldg(sc + p.xs_h + p.xs_w);
                    a[c] = p.round_tf32 ? rna_tf32(acc) : acc;
                }
            }
        }
        const uint32_t slots = (uint32_t)p.CP / 4;                 // 8
        float4* dst = reinterpret_cast<float4*>(out) + (size_t)base * slots;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t owner = 4 * k + (lane >> 3), slot = lane & 7;
            const float r0 = __shfl_sync(0xffffffffu, a[0], owner), r1 = __shfl_sync(0xffffffffu, a[1], owner);
            const float r2 = __shfl_sync(0xffffffffu, a[2], owner), r3 = __shfl_sync(0xffffffffu, a[3], owner);
            if (base + owner < pixels)
                dst[owner * slots + slot] = slot == 0 ? make_float4(r0, r1, r2, r3) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}

// Adjoint in gather form: dx[b, c, y, x] = sum over the crops q of image b, over output rows i with a bilinear foot on y and
// output columns j with a foot on x:  wy(i, y) * wx(j, x) * dy[q, c, i, j].  Output coordinate -> source coordinate is affine
// and monotone (iy = ay + by * i), so the rows with a foot on y are the i with floor(iy) in {y - 1, y}: a contiguous range
// found by inverting the map.  One thread per (b, y, x); the channels share the weights.
__global__ void __launch_bounds__(256)
crop_gather_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, const CropParams p,
                       int64_t ds_n, int64_t ds_c, int64_t ds_h, int64_t ds_w) {
    const int B = p.Q / p.num_crops;
    const int64_t total = (int64_t)B * p.H * p.W;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int xx = (int)(idx % p.W);
        const int yy = (int)((idx / p.W) % p.H);
        const int b = (int)(idx / ((int64_t)p.W * p.H));
        float acc[4] = {0.f, 0.f, 0.f, 0.f};          // C <= 4
        for (int k = 0; k < p.num_crops; ++k) {
            const int q = b * p.num_crops + k;
            const float fl = __ldg(p.flip + q), sx = __ldg(p.scale + 2 * q), sy = __ldg(p.scale + 2 * q + 1);
            const float ox = __ldg(p.offset + 2 * q), oy = __ldg(p.offset + 2 * q + 1);
            // source coordinate of output index t: c(t) = ((lin(t) * s + o + 1) * N - 1) / 2, lin(t) ~ -1 + 2 t / (S - 1):
            // bracket the indices whose foot can touch this pixel generously, then test each exactly
            const float step = 2.f / (float)(p.S - 1);
            const float ay = ((oy - sy + 1.f) * (float)p.H - 1.f) * 0.5f, by = sy * step * (float)p.H * 0.5f;
            const float axs = fl * sx;
            const float ax = ((ox - axs + 1.f) * (float)p.W - 1.f) * 0.5f, bx = axs * step * (float)p.W * 0.5f;
            int i0, i1, j0, j1;
            if (by > 1e-12f) { i0 = (int)floorf(((float)yy - 1.f - ay) / by) - 1; i1 = (int)ceilf(((float)yy + 1.f - ay) / by) + 1; }
            else { i0 = 0; i1 = p.S - 1; }
            if (fabsf(bx) > 1e-12f) {
                const float ja = ((float)xx - 1.f - ax) / bx, jb = ((float)xx + 1.f - ax) / bx;
                j0 = (int)floorf(fminf(ja, jb)) - 1; j1 = (int)ceilf(fmaxf(ja, jb)) + 1;
            } else { j0 = 0; j1 = p.S - 1; }
            i0 = max(i0, 0); i1 = min(i1, p.S - 1); j0 = max(j0, 0); j1 = min(j1, p.S - 1);
            if (i0 > i1 || j0 > j1) continue;
            const float* dq = dy + (int64_t)q * ds_n;
            for (int i = i0; i <= i1; ++i) {
                const float gy = crop_lin(i, p.S) * sy + oy;
                const float iy = ((gy + 1.f) * (float)p.H - 1.f) * 0.5f;
                const float fy = floorf(iy);
                const int y0 = (int)fy;
                float wy;
                if (y0 == yy) wy = 1.f - (iy - fy);
                else if (y0 + 1 == yy) wy = iy - fy;
                else continue;
                for (int j = j0; j <= j1; ++j) {
                    const float gx = (crop_lin(j, p.S) * fl) * sx + ox;
                    const float ix = ((gx + 1.f) * (float)p.W - 1.f) * 0.5f;
                    const float fx = floorf(ix);
                    const int x0 = (int)fx;
                    float wx;
                    if (x0 == xx) wx = 1.f - (ix - fx);
                    else if (x0 + 1 == xx) wx = ix - fx;
                    else continue;
                    const float w = wy * wx;
                    const float* d = dq + (int64_t)i * ds_h + (int64_t)j * ds_w;
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (c < p.C) acc[c] += w * __ldg(d + (int64_t)c * ds_c);
                }
            }
        }
        for (int c = 0; c < p.C; ++c) dx[((int64_t)b * p.C + c) * p.H * p.W + (int64_t)yy * p.W + xx] = acc[c];
    }
}

static inline unsigned grid_1d(int64_t work, int threads, int per_sm) {
    int64_t blocks = (work + threads - 1) / threads;
    const int64_t cap = (int64_t)sm_count() * per_sm;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace sae

using namespace sae;

static int adam_launch(float* const* p_ptrs, const float* const* g_ptrs, const int64_t* offsets, const int64_t* sizes, int n,
                       float* exp_avg, float* exp_avg_sq, float* steps, float lr, float beta1, float beta2, float eps,
                       float grad_scale, const unsigned long long* skip, void* stream) {
    if (n == 0) return SAE_OK;
    if (!p_ptrs || !g_ptrs || !offsets || !sizes || !exp_avg || !exp_avg_sq || !steps || n < 0)
        return fail(SAE_E_INVALID, "adam_step: bad arguments");
    if (!(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f))
        return fail(SAE_E_INVALID, "adam_step: betas must lie in [0, 1) and eps must be >= 0");
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(48, (unsigned)n);
    adam_kernel<<<grid, 256, 0, st>>>(p_ptrs, g_ptrs, offsets, sizes, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, grad_scale,
                                      skip);
    int rc = check_launch("adam_step");
    if (rc) return rc;
    adam_advance_kernel<<<(n + 255) / 256, 256, 0, st>>>(g_ptrs, steps, n, skip);
    return check_launch("adam_advance");
}

extern "C" int sae_adam_step(float* const* p_ptrs, const float* const* g_ptrs, const int64_t* offsets, const int64_t* sizes,
                             int n, float* exp_avg, float* exp_avg_sq, float* steps, float lr, float beta1, float beta2,
                             float eps, float grad_scale, void* stream) {
    return adam_launch(p_ptrs, g_ptrs, offsets, sizes, n, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, grad_scale, nullptr,
                       stream);
}

extern "C" int sae_adam_step_guarded(float* const* p_ptrs, const float* const* g_ptrs, const int64_t* offsets,
                                     const int64_t* sizes, int n, float* exp_avg, float* exp_avg_sq, float* steps, float lr,
                                     float beta1, float beta2, float eps, float grad_scale, const unsigned long long* skip,
                                     void* stream) {
    if (!skip && n != 0) return fail(SAE_E_INVALID, "adam_step_guarded: null skip pointer");
    return adam_launch(p_ptrs, g_ptrs, offsets, sizes, n, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, grad_scale, skip,
                       stream);
}

static int crop_params(CropParams& p, const float* flip, const float* scale, const float* offset, int Q, int num_crops, int C,
                       int H, int W, int S, int CP, const char* who) {
    if (!flip || !scale || !offset) return fail(SAE_E_INVALID, "%s: null crop parameters", who);
    if (Q < 0 || num_crops <= 0 || Q % num_crops != 0 || C <= 0 || C > 4 || H <= 0 || W <= 0 || S < 2)
        return fail(SAE_E_INVALID, "%s: bad geometry (1..4 channels, target size >= 2)", who);
    if (CP < C || CP % 4 != 0) return fail(SAE_E_INVALID, "%s: padded channel count must be a multiple of 4 and >= C", who);
    p.flip = flip; p.scale = scale; p.offset = offset;
    p.Q = Q; p.num_crops = num_crops; p.C = C; p.H = H; p.W = W; p.S = S; p.CP = CP;
    return SAE_OK;
}

extern "C" int sae_crop_gather(const float* x, const float* flip, const float* scale, const float* offset, float* out,
                               int Q, int num_crops, int C, int H, int W, int S, int CP,
                               int64_t xs_n, int64_t xs_c, int64_t xs_h, int64_t xs_w, int round_tf32, void* stream) {
    if (Q == 0) return SAE_OK;
    CropParams p;
    int rc = crop_params(p, flip, scale, offset, Q, num_crops, C, H, W, S, CP, "crop_gather");
    if (rc) return rc;
    if (!x || !out || (reinterpret_cast<uintptr_t>(out) & 15)) return fail(SAE_E_INVALID, "crop_gather: null / unaligned pointer");
    if ((int64_t)Q * S * S * (CP / 4) >= ((int64_t)1 << 32)) return fail(SAE_E_UNSUPPORTED, "crop_gather: more than 2^32 output slots");
    if (CP != 32) return fail(SAE_E_UNSUPPORTED, "crop_gather: the padded width must be 32 channels (one 128-byte row per pixel)");
    p.xs_n = xs_n; p.xs_c = xs_c; p.xs_h = xs_h; p.xs_w = xs_w; p.round_tf32 = round_tf32;
    crop_gather_kernel<<<grid_1d((int64_t)Q * S * S, 256, 8), 256, 0, (cudaStream_t)stream>>>(x, out, p);
    return check_launch("crop_gather");
}

extern "C" int sae_crop_gather_backward(const float* dy, const float* flip, const float* scale, const float* offset, float* dx,
                                        int Q, int num_crops, int C, int H, int W, int S,
                                        int64_t ds_n, int64_t ds_c, int64_t ds_h, int64_t ds_w, void* stream) {
    if (Q == 0) return SAE_OK;
    CropParams p;
    int rc = crop_params(p, flip, scale, offset, Q, num_crops, C, H, W, S, 4, "crop_gather_backward");
    if (rc) return rc;
    if (!dy || !dx) return fail(SAE_E_INVALID, "crop_gather_backward: null pointer");
    p.xs_n = p.xs_c = p.xs_h = p.xs_w = 0; p.round_tf32 = 0;
    crop_gather_bwd_kernel<<<grid_1d((int64_t)(Q / num_crops) * H * W, 256, 16), 256, 0, (cudaStream_t)stream>>>(
        dy, dx, p, ds_n, ds_c, ds_h, ds_w);
    return check_launch("crop_gather_backward");
}
