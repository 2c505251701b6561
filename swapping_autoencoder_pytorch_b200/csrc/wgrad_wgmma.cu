// Weight gradient of the convolution on the Hopper tensor cores (wgmma, tf32 inputs, fp32 accumulators in registers).
//
//   dW[o, (tap, c)] += sum_{pixels (n,p,q)}  dy[n,p,q,o] * x[n, p*st - pad_t + r, q*st - pad_l + s, c]
//
// GEMM view: M = out channels (128 per CTA), N = (tap, in channel) columns (128 per CTA), K = pixels (32 per stage).
// In NHWC both operands are MN-major (channels contiguous, the reduction runs over pixels), and wgmma reads tf32 operands
// from shared memory K-major only.  So:
//   * A (dy) goes to wgmma from REGISTERS, which carry no major-ness: each warp loads its m16 x k8 fragments straight out of
//     the pixel-major dy tile (row stride 136 floats: conflict-free);
//   * B (the gathered x) is transposed once per stage into the K-major 128-byte-swizzled layout: every thread moves 16-byte
//     pieces (4 pixels of one column), consecutive lanes take consecutive columns, so both the reads and the swizzled
//     16-byte writes are free of bank conflicts;
//   * both tiles arrive by cp.async (the x tile gathered per pixel, out-of-range taps zero-filled), two stages, two CTAs
//     per SM: one CTA transposes and loads while the other's wgmma run;
//   * grid = (out-channel tiles, column tiles, pixel splits); partial tiles are reduced into dW with fp32 atomics (dW is
//     zero-initialised by the caller).  Style-modulated mode (p.img_pix > 0): chunks never straddle images and the drain
//     forms dW += s[n, c] G_n and ds[n, c] += sum_{o, tap} W[o, tap, c] G_n from the unscaled input (ds summed over the
//     CTA's 128 rows in shared memory, one atomic per column).
// Operands are rounded to TF32 (cvt.rna) on their way into the fragments / the transposed tile, as in the mma.sync kernel.
// Split-TF32 (SPLIT = true, the fp32 precision mode): every operand is split into hi = rna_tf32(v), lo = rna_tf32(v - hi); the
// dy fragments in registers, the gathered x into a hi and a lo K-major tile (+16 KB), and each k8 step issues
// dy_lo x_hi + dy_hi x_lo + dy_hi x_hi.  The tensor core's accumulation rounds toward zero, so these wgmma accumulate one stage
// into partial sums (scale-d = 0 on the first) that are added into the accumulators with round-to-nearest fp32 adds; with the
// second accumulator set the kernel runs one CTA per SM.
#include "tc_common.cuh"

namespace sae {

constexpr int WGR_THREADS = 256;                  // two warpgroups: output-channel rows [0, 64) and [64, 128)
constexpr int WGR_BK = 32;                        // pixels per stage
constexpr int WGR_LD = 128 + 8;                   // row stride (floats) of the pixel-major staging tiles
constexpr int WGR_TILE = WGR_BK * WGR_LD * 4;     // bytes of one pixel-major tile
constexpr int WGR_BT = 128 * WGR_BK * 4;          // the K-major swizzled B tile: 128 rows x 128 bytes = 16 KB
template <bool SPLIT>
constexpr size_t wgr_smem() { return (size_t)(SPLIT ? 2 : 1) * WGR_BT + 4 * (size_t)WGR_TILE + 1024; }

__device__ __forceinline__ void cp_async16_wg(uint32_t s, const void* gmem, bool pred) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(pred ? 16 : 0));
}

template <bool SPLIT>
__global__ void __launch_bounds__(WGR_THREADS, SPLIT ? 1 : 2)
wgrad_wg_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dw, const WgradParams p) {
    constexpr int BT_BYTES = (SPLIT ? 2 : 1) * WGR_BT;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;       // SWIZZLE_128B needs 1024-byte alignment
    uint8_t* smem_gen = smem_raw + (base - smem_u32(smem_raw));
    uint8_t* bt = smem_gen;                                            // K-major B tile (SPLIT: hi, then lo)
    const uint32_t bt_s = base;
    float* tiles = reinterpret_cast<float*>(smem_gen + BT_BYTES);      // [stage][A, B][WGR_BK][WGR_LD]
    const uint32_t tiles_s = base + BT_BYTES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const int o0 = blockIdx.x * 128, n0 = blockIdx.y * 128;
    const int64_t pix0 = (int64_t)blockIdx.z * p.chunk;
    const int64_t pix1 = pix0 + p.chunk < p.Mpix ? pix0 + p.chunk : p.Mpix;
    const int KB = (int)((pix1 - pix0 + WGR_BK - 1) / WGR_BK);

    // loader: this thread always serves channel quad cq of both operands, pixel rows (tid >> 5) + 8 j of the stage
    const int cq = tid & 31;
    const int oa = o0 + cq * 4;
    const bool a_ok = oa < p.Ko;
    const int nb = n0 + cq * 4;
    const bool b_ok = nb < p.Ncol;
    const int tap = b_ok ? nb / p.C : 0;
    const int bc = nb - tap * p.C, br = tap / p.S, bs = tap - br * p.S;
    auto load_stage = [&](int stage, int kb) {
        const uint32_t as = tiles_s + (uint32_t)(2 * stage) * WGR_TILE, bsm = as + WGR_TILE;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int kp = (tid >> 5) + 8 * j;
            const int64_t pix = pix0 + (int64_t)kb * WGR_BK + kp;
            const bool ok = pix < pix1;
            cp_async16_wg(as + (uint32_t)(kp * WGR_LD + cq * 4) * 4u, (ok && a_ok) ? dy + pix * p.Ko + oa : dy, ok && a_ok);
            const float* gp = x;
            bool okb = ok && b_ok;
            if (okb) {
                const int q = (int)(pix % p.Q);
                const int64_t r2 = pix / p.Q;
                const int pp = (int)(r2 % p.P);
                const int64_t ni = r2 / p.P;
                const int iy = pp * p.stride - p.pad_t + br, ix = q * p.stride - p.pad_l + bs;
                okb = iy >= 0 && ix >= 0 && iy < p.H && ix < p.W;
                if (okb) gp = x + ((ni * p.H + iy) * (int64_t)p.W + ix) * p.C + bc;
            }
            cp_async16_wg(bsm + (uint32_t)(kp * WGR_LD + cq * 4) * 4u, gp, okb);
        }
    };

    float acc[64];
    float part[SPLIT ? 64 : 1];                                        // split-TF32: the current stage's sums
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    if (KB > 0) load_stage(0, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const int r0 = wg * 64 + (warp & 3) * 16 + g;                      // this thread's A-fragment rows r0, r0 + 8
    for (int kb = 0; kb < KB; ++kb) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                      // stage kb has landed; the previous stage's wgmma (waited below) are done
        if (kb + 1 < KB) load_stage((kb + 1) & 1, kb + 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        const float* at = tiles + (size_t)(2 * (kb & 1)) * (WGR_TILE / 4);
        const float* bsrc = at + WGR_TILE / 4;
        if constexpr (SPLIT) {
            // B_hi, B_lo: the same transpose, two tiles
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) {
                const int idx = tid + WGR_THREADS * qd;
                const int n = idx & 127, c4 = idx >> 7;
                uint32_t h[4], l[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) split_tf32(bsrc[(4 * c4 + u) * WGR_LD + n], h[u], l[u]);
                const int off = n * 128 + ((c4 ^ (n & 7)) << 4);
                *reinterpret_cast<uint4*>(bt + off) = make_uint4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<uint4*>(bt + WGR_BT + off) = make_uint4(l[0], l[1], l[2], l[3]);
            }
            uint32_t ahi[4][4], alo[4][4];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const float* ap = at + (ks * 8 + t) * WGR_LD + r0;
                split_tf32(ap[0], ahi[ks][0], alo[ks][0]);
                split_tf32(ap[8], ahi[ks][1], alo[ks][1]);
                split_tf32(ap[4 * WGR_LD], ahi[ks][2], alo[ks][2]);
                split_tf32(ap[4 * WGR_LD + 8], ahi[ks][3], alo[ks][3]);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            const uint64_t db = make_wgmma_desc_sw128(bt_s), dbl = make_wgmma_desc_sw128(bt_s + WGR_BT);
            wgmma_fence();
            wgmma_tf32_n128_rs<0>(part, alo[0], db);
            wgmma_tf32_n128_rs<1>(part, ahi[0], dbl);
            wgmma_tf32_n128_rs<1>(part, ahi[0], db);
#pragma unroll
            for (int ks = 1; ks < 4; ++ks) {
                wgmma_tf32_n128_rs<1>(part, alo[ks], db + (uint64_t)(ks * 2));
                wgmma_tf32_n128_rs<1>(part, ahi[ks], dbl + (uint64_t)(ks * 2));
                wgmma_tf32_n128_rs<1>(part, ahi[ks], db + (uint64_t)(ks * 2));
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] += part[i];
        } else {
            // B: pixel-major [32][136] -> K-major swizzled [128 rows][32 pixels]
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) {
                const int idx = tid + WGR_THREADS * qd;
                const int n = idx & 127, c4 = idx >> 7;                    // column n, pixels 4 c4 .. 4 c4 + 3
                float4 v;
                v.x = rna_tf32(bsrc[(4 * c4 + 0) * WGR_LD + n]);
                v.y = rna_tf32(bsrc[(4 * c4 + 1) * WGR_LD + n]);
                v.z = rna_tf32(bsrc[(4 * c4 + 2) * WGR_LD + n]);
                v.w = rna_tf32(bsrc[(4 * c4 + 3) * WGR_LD + n]);
                *reinterpret_cast<float4*>(bt + n * 128 + ((c4 ^ (n & 7)) << 4)) = v;
            }
            // A: m16 x k8 fragments of dy^T (rows = out channels, columns = pixels) from the pixel-major tile
            uint32_t a[4][4];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const float* ap = at + (ks * 8 + t) * WGR_LD + r0;
                a[ks][0] = __float_as_uint(rna_tf32(ap[0]));
                a[ks][1] = __float_as_uint(rna_tf32(ap[8]));
                a[ks][2] = __float_as_uint(rna_tf32(ap[4 * WGR_LD]));
                a[ks][3] = __float_as_uint(rna_tf32(ap[4 * WGR_LD + 8]));
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> visible to wgmma
            __syncthreads();
            const uint64_t db = make_wgmma_desc_sw128(bt_s);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) wgmma_tf32_n128_rs(acc, a[ks], db + (uint64_t)(ks * 2));   // +32 bytes along K
            wgmma_commit();
            wgmma_wait<0>();
        }
    }

    // accumulator fragment: rows o0 + r0 (+ 8), columns n0 + 8 j + 2 t + {0, 1}
    const int orow = o0 + r0;
    if (p.img_pix > 0) {
        const int img = (int)(pix0 / p.img_pix);
        // ds: each warp's column sums over its 16 rows (shuffles) land in dsp[warp][column]; then one thread per column adds the
        // 8 warps in a fixed order and issues ONE atomic per column and CTA (few, order-stable contributions per ds element)
        __syncthreads();                                              // the staging tiles are free: every wgmma has retired
        float* dsp = tiles;                                           // [8 warps][128 columns]
        for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int n = n0 + 8 * j + 2 * t + u;
                const bool nok = n < p.Ncol;
                const int c = nok ? n % p.C : 0;
                const float sc = nok ? __ldg(p.mod_s + (int64_t)img * p.C + c) : 0.f;
                float dsum = 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int o = orow + 8 * h;
                    if (o >= p.Ko || !nok) continue;
                    const float v = acc[4 * j + 2 * h + u];
                    dsum += v * __ldg(p.mod_w + (int64_t)o * p.Ncol + n);
                    atomicAdd(dw + (int64_t)o * p.Ncol + n, v * sc);
                }
                // the 8 lanes of a column (g = 0..7) share n
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 4);
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 8);
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 16);
                if (g == 0) dsp[warp * 128 + 8 * j + 2 * t + u] = dsum;
            }
        __syncthreads();
        if (tid < 128 && n0 + tid < p.Ncol) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += dsp[w * 128 + tid];
            atomicAdd(p.mod_ds + (int64_t)img * p.C + (n0 + tid) % p.C, v);
        }
        return;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int n = n0 + 8 * j + 2 * t;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int o = orow + 8 * h;
            if (o >= p.Ko) continue;
            if (n < p.Ncol) atomicAdd(dw + (int64_t)o * p.Ncol + n, acc[4 * j + 2 * h]);
            if (n + 1 < p.Ncol) atomicAdd(dw + (int64_t)o * p.Ncol + n + 1, acc[4 * j + 2 * h + 1]);
        }
    }
}

bool wgrad_wg_eligible(const sae_conv_geom* g) { return g->K % 4 == 0 && g->C % 4 == 0; }

template <bool SPLIT>
static int wgrad_wg_launch_t(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st) {
    constexpr size_t smem = wgr_smem<SPLIT>();
    static bool attr_done = false;
    if (!attr_done) {
        SAE_CUDA_TRY(cudaFuncSetAttribute(wgrad_wg_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    dim3 grid((unsigned)((p.Ko + 127) / 128), (unsigned)((p.Ncol + 127) / 128), splits);
    wgrad_wg_kernel<SPLIT><<<grid, WGR_THREADS, smem, st>>>(dy, x, dw, p);
    return check_launch("wgrad_wg");
}

int wgrad_wg_launch(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st, bool split) {
    return split ? wgrad_wg_launch_t<true>(dy, x, dw, p, splits, st) : wgrad_wg_launch_t<false>(dy, x, dw, p, splits, st);
}

}  // namespace sae
