// Generic implicit-GEMM convolution on NHWC fp32 with mma.sync TF32 (m16n8k8) — the shape-complete
// kernel of the conv family (any stride / padding / channel count, forward, data-gradient incl.
// transposed convolution, weight-gradient).  The wgmma kernels take over the shapes that carry the
// FLOPs (SURVEY.md Appendix A): conv_wgmma.cu the forward and data-gradient passes, wgrad_wgmma.cu the
// weight gradients whose channel counts are multiples of 4; this file covers what they cannot tile —
// Cin = 3 (FromRGB), Cout = 3 / 1 (ToRGB, final linears), 7x7 / 3x3 maps, fractional strides — and is
// the impl = 1 reference path.
//
// fprop / dgrad share one "gather GEMM":  C[m, n] = sum_k A[m, k] * B[n, k]
//   m = output pixel (n_img, oy, ox), k = (tap r,s ; source channel c), A gathered on the fly:
//   iy = (oy*SY + OFFY + r*DY) / DIV  (only if divisible and in range), same in x.
//   fprop: SY = stride, DY = +1, OFF = -pad, DIV = 1;  dgrad: SY = 1, DY = -1, OFF = +pad, DIV = stride.
// wgrad:  dW[o, (r,s,c)] += sum_pixels dy[pixel, o] * x_gathered[pixel, (r,s,c)], split over pixels,
//   fp32 atomics into dW.
// Operands are rounded to TF32 (cvt.rna) when fragments are loaded, accumulation is fp32.
// Split-TF32 (SPLIT = true, the fp32 precision mode): the activation operands are split into hi = rna_tf32(v),
// lo = rna_tf32(v - hi) in registers, the gather kernel's filter arrives as the pair (wmat = hi, wlo = lo), and every
// fragment pair issues three mma (lo*hi + hi*lo + hi*hi).
#include "conv_internal.cuh"

namespace sae {

constexpr int BM = 128, BK = 32, LDS_K = BK + 4, STAGES = 3, NTHREADS = 256;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool pred) {
    uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    int sz = pred ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

__device__ __forceinline__ uint32_t to_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// split-TF32 product of one fragment pair, acc += a b with a = ah + al, b = bh + bl.  The tensor core adds into its
// accumulator rounding toward zero, a bias that over a long K reaches ~1e-5 relative; so the three products go into a fresh
// fragment and reach acc through round-to-nearest fp32 adds.
__device__ __forceinline__ void mma_tf32_3x(float (&acc)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                            const uint32_t (&bh)[2], const uint32_t (&bl)[2]) {
    float t[4];
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=f"(t[0]), "=f"(t[1]), "=f"(t[2]), "=f"(t[3])
                 : "r"(al[0]), "r"(al[1]), "r"(al[2]), "r"(al[3]), "r"(bh[0]), "r"(bh[1]), "f"(0.f));
    mma_tf32(t, ah, bl);
    mma_tf32(t, ah, bh);
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] += t[q];
}

// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------ deterministic slot reduction
// dst[i] (+)= ws[0][i] + ws[1][i] + ... in slot order: the reduction behind every _det entry point
__global__ void __launch_bounds__(256)
det_reduce_kernel(float* __restrict__ dst, const float* __restrict__ ws, int64_t slots, int64_t n, int accumulate, int round_tf32) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float v = ws[i];
        for (int64_t s = 1; s < slots; ++s) v += ws[s * n + i];
        if (accumulate) v = dst[i] + v;
        dst[i] = round_tf32 ? rna_tf32(v) : v;
    }
}

int det_reduce(float* dst, const float* ws, int64_t slots, int64_t n, bool accumulate, int round_tf32, cudaStream_t st) {
    if (n == 0 || slots == 0) return SAE_OK;
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)DET_SMS * 16) blocks = (int64_t)DET_SMS * 16;
    det_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(dst, ws, slots, n, accumulate ? 1 : 0, round_tf32);
    return check_launch("det_reduce");
}

// ------------------------------------------------------------------------------------------------
// DET (split-K only): `out` is the workspace, one [M, Ncol] slab per K split (slot = blockIdx.z), written with plain stores
template <int BN, bool VEC, bool SPLIT, bool DET>
__global__ void __launch_bounds__(NTHREADS)
conv_gather_kernel(const float* __restrict__ src, const float* __restrict__ wmat, float* __restrict__ out,
                   GatherParams p, EpiParams e, const float* __restrict__ wlo) {
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                               // [STAGES][BM][LDS_K]
    float* Bs = smem + STAGES * BM * LDS_K;         // [STAGES][BN][LDS_K]
    float* Bl = Bs + STAGES * BN * LDS_K;           // SPLIT: [STAGES][BN][LDS_K], the filter's low halves

    constexpr int WARPS_N = BN / 32;
    constexpr int WARPS_M = 8 / WARPS_N;
    constexpr int WM = BM / WARPS_M;                // rows per warp
    constexpr int MT = WM / 16;                     // m16 tiles per warp
    constexpr int NT = 4;                           // n8 tiles per warp (32 columns)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp / WARPS_N, wn = warp % WARPS_N;
    const int g = lane >> 2, t = lane & 3;

    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int KB_total = (p.K + BK - 1) / BK;
    // split-K (gridDim.z > 1, small-M GEMMs such as the style / head linears): this CTA reduces k-blocks
    // [kb_begin, kb_begin + KB) and adds its partial tile to the zero-initialised output with fp32 atomics
    const int kb_per = (KB_total + (int)gridDim.z - 1) / (int)gridDim.z;
    const int kb_begin = (int)blockIdx.z * kb_per;
    const int KB = max(0, min(kb_per, KB_total - kb_begin));
    const bool split = gridDim.z > 1;

    // per-thread row bookkeeping for the vector loader: rows (tid>>3) + j*32, j = 0..3
    int row_oy[4], row_ox[4];
    int64_t row_base[4];
    bool row_ok[4];
    if (VEC) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int64_t m = m0 + (tid >> 3) + j * 32;
            row_ok[j] = m < p.M;
            int64_t mm = row_ok[j] ? m : 0;
            int ox = (int)(mm % p.OW);
            int64_t q = mm / p.OW;
            int oy = (int)(q % p.OH);
            int64_t ni = q / p.OH;
            row_oy[j] = oy * p.SY + p.OFFY;
            row_ox[j] = ox * p.SY + p.OFFX;
            row_base[j] = ni * (int64_t)p.IH * p.IW;
        }
    }

    auto load_stage = [&](int stage, int kb_rel) {
        const int kb = kb_begin + kb_rel;
        float* as = As + stage * BM * LDS_K;
        float* bs = Bs + stage * BN * LDS_K;
        float* bl = Bl + stage * BN * LDS_K;
        if (VEC) {
            const int kq = tid & 7;
            const int k = kb * BK + kq * 4;
            const bool kok = k < p.K;
            int tap = kok ? k / p.Cs : 0;
            int c = k - tap * p.Cs;
            int r = tap / p.S, s = tap - r * p.S;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int row = (tid >> 3) + j * 32;
                int iy = row_oy[j] + r * p.DY, ix = row_ox[j] + s * p.DY;
                bool ok = kok && row_ok[j] && iy >= 0 && ix >= 0;
                if (p.DIV > 1) {
                    ok = ok && (iy % p.DIV == 0) && (ix % p.DIV == 0);
                    iy /= p.DIV; ix /= p.DIV;
                }
                ok = ok && iy < p.IH && ix < p.IW;
                const float* gp = ok ? src + (row_base[j] + (int64_t)iy * p.IW + ix) * p.Cs + c : src;
                cp_async16(as + row * LDS_K + kq * 4, gp, ok);
            }
#pragma unroll
            for (int j = 0; j < BN / 32; ++j) {
                int row = (tid >> 3) + j * 32;
                int n = n0 + row;
                bool ok = kok && n < p.Ncol;
                const float* gp = ok ? wmat + (int64_t)n * p.K + k : wmat;
                cp_async16(bs + row * LDS_K + kq * 4, gp, ok);
                if constexpr (SPLIT) cp_async16(bl + row * LDS_K + kq * 4, ok ? wlo + (int64_t)n * p.K + k : wlo, ok);
            }
        } else {
            // scalar path (channel counts that are not multiples of 4): plain loads
            for (int f = tid; f < BM * BK; f += NTHREADS) {
                int row = f >> 5, kk = f & 31;
                int k = kb * BK + kk;
                int64_t m = m0 + row;
                float v = 0.f;
                if (k < p.K && m < p.M) {
                    int tap = k / p.Cs, c = k - tap * p.Cs;
                    int r = tap / p.S, s = tap - r * p.S;
                    int ox = (int)(m % p.OW);
                    int64_t q = m / p.OW;
                    int oy = (int)(q % p.OH);
                    int64_t ni = q / p.OH;
                    int iy = oy * p.SY + p.OFFY + r * p.DY, ix = ox * p.SY + p.OFFX + s * p.DY;
                    bool ok = iy >= 0 && ix >= 0;
                    if (p.DIV > 1) {
                        ok = ok && (iy % p.DIV == 0) && (ix % p.DIV == 0);
                        iy /= p.DIV; ix /= p.DIV;
                    }
                    ok = ok && iy < p.IH && ix < p.IW;
                    if (ok) v = __ldg(src + ((ni * p.IH + iy) * (int64_t)p.IW + ix) * p.Cs + c);
                }
                as[row * LDS_K + kk] = v;
            }
            for (int f = tid; f < BN * BK; f += NTHREADS) {
                int row = f >> 5, kk = f & 31;
                int k = kb * BK + kk, n = n0 + row;
                float v = 0.f;
                if (k < p.K && n < p.Ncol) v = __ldg(wmat + (int64_t)n * p.K + k);
                bs[row * LDS_K + kk] = v;
                if constexpr (SPLIT) bl[row * LDS_K + kk] = (k < p.K && n < p.Ncol) ? __ldg(wlo + (int64_t)n * p.K + k) : 0.f;
            }
        }
    };

    float acc[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KB) load_stage(s, s);
        cp_async_commit();
    }
    for (int kb = 0; kb < KB; ++kb) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            int nk = kb + STAGES - 1;
            if (nk < KB) load_stage(nk % STAGES, nk);
            cp_async_commit();
        }
        const float* as = As + (kb % STAGES) * BM * LDS_K + (wm * WM) * LDS_K;
        const float* bs = Bs + (kb % STAGES) * BN * LDS_K + (wn * 32) * LDS_K;
        if constexpr (SPLIT) {
            const float* bl = Bl + (kb % STAGES) * BN * LDS_K + (wn * 32) * LDS_K;
#pragma unroll
            for (int ks = 0; ks < BK / 8; ++ks) {
                uint32_t ah[MT][4], al[MT][4], bh[NT][2], blo[NT][2];
#pragma unroll
                for (int i = 0; i < MT; ++i) {
                    const float* a = as + (i * 16 + g) * LDS_K + ks * 8 + t;
                    split_tf32(a[0], ah[i][0], al[i][0]);
                    split_tf32(a[8 * LDS_K], ah[i][1], al[i][1]);
                    split_tf32(a[4], ah[i][2], al[i][2]);
                    split_tf32(a[8 * LDS_K + 4], ah[i][3], al[i][3]);
                }
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    const int o = (j * 8 + g) * LDS_K + ks * 8 + t;
                    bh[j][0] = __float_as_uint(bs[o]);
                    bh[j][1] = __float_as_uint(bs[o + 4]);
                    blo[j][0] = __float_as_uint(bl[o]);
                    blo[j][1] = __float_as_uint(bl[o + 4]);
                }
#pragma unroll
                for (int i = 0; i < MT; ++i)
#pragma unroll
                    for (int j = 0; j < NT; ++j) mma_tf32_3x(acc[i][j], ah[i], al[i], bh[j], blo[j]);
            }
            continue;
        }
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) {
            uint32_t af[MT][4], bf[NT][2];
#pragma unroll
            for (int i = 0; i < MT; ++i) {
                const float* a = as + (i * 16 + g) * LDS_K + ks * 8 + t;
                af[i][0] = to_tf32(a[0]);
                af[i][1] = to_tf32(a[8 * LDS_K]);
                af[i][2] = to_tf32(a[4]);
                af[i][3] = to_tf32(a[8 * LDS_K + 4]);
            }
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const float* b = bs + (j * 8 + g) * LDS_K + ks * 8 + t;
                bf[j][0] = to_tf32(b[0]);
                bf[j][1] = to_tf32(b[4]);
            }
#pragma unroll
            for (int i = 0; i < MT; ++i)
#pragma unroll
                for (int j = 0; j < NT; ++j) mma_tf32(acc[i][j], af[i], bf[j]);
        }
    }
    cp_async_wait<0>();

    // epilogue (split-K runs only with the plain epilogue; launch_gather applies round_tf32 to the summed output)
    if (split) {
        float* const outz = DET ? out + (int64_t)blockIdx.z * p.M * p.Ncol : out;
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                int64_t m = m0 + wm * WM + i * 16 + g + h * 8;
                if (m >= p.M) continue;
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        int col = n0 + wn * 32 + j * 8 + 2 * t + u;
                        if (col < p.Ncol) drain_add<DET>(outz + m * p.Ncol + col, acc[i][j][h * 2 + u]);
                    }
            }
        return;
    }
    if (p.Ncol % 4 == 0) {
        // stage the tile in shared memory (the pipeline buffers are free now) and write whole rows with float4 stores:
        // the m16n8 fragment layout would otherwise scatter 8-byte stores over 8 rows per instruction
        constexpr int LDC = BN + 4;
        __syncthreads();
        float* cs = smem;
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = wm * WM + i * 16 + g + h * 8;
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    const int c = wn * 32 + j * 8 + 2 * t;
                    *reinterpret_cast<float2*>(cs + r * LDC + c) = make_float2(acc[i][j][h * 2], acc[i][j][h * 2 + 1]);
                }
            }
        __syncthreads();
        constexpr int C4 = BN / 4;
        for (int f = tid; f < BM * C4; f += NTHREADS) {
            const int r = f / C4, c4 = f - r * C4;
            const int64_t m = m0 + r;
            const int col = n0 + c4 * 4;
            if (m >= p.M || col >= p.Ncol) continue;
            float4 v = *reinterpret_cast<const float4*>(cs + r * LDC + c4 * 4);
            v.x = apply_epi(e, v.x, m, col, p.Ncol);
            v.y = apply_epi(e, v.y, m, col + 1, p.Ncol);
            v.z = apply_epi(e, v.z, m, col + 2, p.Ncol);
            v.w = apply_epi(e, v.w, m, col + 3, p.Ncol);
            *reinterpret_cast<float4*>(out + m * p.Ncol + col) = v;
        }
        return;
    }
    const bool even = (p.Ncol % 2 == 0);
#pragma unroll
    for (int i = 0; i < MT; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int64_t m = m0 + wm * WM + i * 16 + g + h * 8;
            if (m >= p.M) continue;
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                int col = n0 + wn * 32 + j * 8 + 2 * t;
                if (col >= p.Ncol) continue;
                float v0 = apply_epi(e, acc[i][j][h * 2 + 0], m, col, p.Ncol);
                float* dst = out + m * p.Ncol + col;
                if (col + 1 < p.Ncol) {
                    float v1 = apply_epi(e, acc[i][j][h * 2 + 1], m, col + 1, p.Ncol);
                    if (even) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
                    else { dst[0] = v0; dst[1] = v1; }
                } else {
                    dst[0] = v0;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
constexpr int LDS_M = 128 + 8;

// DET: dw is the workspace's dW region, one [Ko, Ncol] slab per pixel split (slot = blockIdx.z), and p.mod_ds its ds region
// (N * C floats per slot, row group = one warp row of 64 output channels: see wgrad_ds_slot)
template <bool VA, bool VB, bool SPLIT, bool DET>
__global__ void __launch_bounds__(NTHREADS)
conv_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dw, WgradParams p) {
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                              // [STAGES][BK][LDS_M]   (k = pixel, m = out channel)
    float* Bs = smem + STAGES * BK * LDS_M;        // [STAGES][BK][LDS_M]   (k = pixel, n = (tap, c))

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;       // 2 x 4 warps, warp tile 64 x 32
    const int g = lane >> 2, t = lane & 3;
    const int o0 = blockIdx.x * 128;
    const int n0 = blockIdx.y * 128;
    const int64_t pix0 = (int64_t)blockIdx.z * p.chunk;
    int64_t pix1 = pix0 + p.chunk;
    if (pix1 > p.Mpix) pix1 = p.Mpix;
    const int KB = (int)((pix1 - pix0 + BK - 1) / BK);

    // vector loader bookkeeping: this thread always serves column quad (tid & 31)
    const int cq = tid & 31;
    int b_tap_r = 0, b_tap_s = 0, b_c = 0;
    bool b_colok = false;
    if (VB) {
        int n = n0 + cq * 4;
        b_colok = n < p.Ncol;
        int tap = b_colok ? n / p.C : 0;
        b_c = n - tap * p.C;
        b_tap_r = tap / p.S;
        b_tap_s = tap - b_tap_r * p.S;
    }

    auto load_stage = [&](int stage, int kb) {
        float* as = As + stage * BK * LDS_M;
        float* bs = Bs + stage * BK * LDS_M;
        if (VA) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int kp = (tid >> 5) + j * 8;
                int64_t pix = pix0 + (int64_t)kb * BK + kp;
                int o = o0 + cq * 4;
                bool ok = pix < pix1 && o < p.Ko;
                const float* gp = ok ? dy + pix * p.Ko + o : dy;
                cp_async16(as + kp * LDS_M + cq * 4, gp, ok);
            }
        } else {
            for (int f = tid; f < BK * 128; f += NTHREADS) {
                int kp = f >> 7, mm = f & 127;
                int64_t pix = pix0 + (int64_t)kb * BK + kp;
                int o = o0 + mm;
                float v = 0.f;
                if (pix < pix1 && o < p.Ko) v = __ldg(dy + pix * p.Ko + o);
                as[kp * LDS_M + mm] = v;
            }
        }
        if (VB) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int kp = (tid >> 5) + j * 8;
                int64_t pix = pix0 + (int64_t)kb * BK + kp;
                bool ok = b_colok && pix < pix1;
                const float* gp = x;
                if (ok) {
                    int q = (int)(pix % p.Q);
                    int64_t r2 = pix / p.Q;
                    int pp = (int)(r2 % p.P);
                    int64_t ni = r2 / p.P;
                    int iy = pp * p.stride - p.pad_t + b_tap_r;
                    int ix = q * p.stride - p.pad_l + b_tap_s;
                    ok = iy >= 0 && ix >= 0 && iy < p.H && ix < p.W;
                    if (ok) gp = x + ((ni * p.H + iy) * (int64_t)p.W + ix) * p.C + b_c;
                }
                cp_async16(bs + kp * LDS_M + cq * 4, gp, ok);
            }
        } else {
            for (int f = tid; f < BK * 128; f += NTHREADS) {
                int kp = f >> 7, nn = f & 127;
                int64_t pix = pix0 + (int64_t)kb * BK + kp;
                int n = n0 + nn;
                float v = 0.f;
                if (pix < pix1 && n < p.Ncol) {
                    int tap = n / p.C, c = n - tap * p.C;
                    int r = tap / p.S, s = tap - r * p.S;
                    int q = (int)(pix % p.Q);
                    int64_t r2 = pix / p.Q;
                    int pp = (int)(r2 % p.P);
                    int64_t ni = r2 / p.P;
                    int iy = pp * p.stride - p.pad_t + r;
                    int ix = q * p.stride - p.pad_l + s;
                    if (iy >= 0 && ix >= 0 && iy < p.H && ix < p.W)
                        v = __ldg(x + ((ni * p.H + iy) * (int64_t)p.W + ix) * p.C + c);
                }
                bs[kp * LDS_M + nn] = v;
            }
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KB) load_stage(s, s);
        cp_async_commit();
    }
    for (int kb = 0; kb < KB; ++kb) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            int nk = kb + STAGES - 1;
            if (nk < KB) load_stage(nk % STAGES, nk);
            cp_async_commit();
        }
        const float* as = As + (kb % STAGES) * BK * LDS_M + wm * 64;
        const float* bs = Bs + (kb % STAGES) * BK * LDS_M + wn * 32;
        if constexpr (SPLIT) {
#pragma unroll
            for (int ks = 0; ks < BK / 8; ++ks) {
                uint32_t ah[4][4], al[4][4], bh[4][2], blo[4][2];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float* a = as + (ks * 8 + t) * LDS_M + i * 16 + g;
                    split_tf32(a[0], ah[i][0], al[i][0]);
                    split_tf32(a[8], ah[i][1], al[i][1]);
                    split_tf32(a[4 * LDS_M], ah[i][2], al[i][2]);
                    split_tf32(a[4 * LDS_M + 8], ah[i][3], al[i][3]);
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float* b = bs + (ks * 8 + t) * LDS_M + j * 8 + g;
                    split_tf32(b[0], bh[j][0], blo[j][0]);
                    split_tf32(b[4 * LDS_M], bh[j][1], blo[j][1]);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) mma_tf32_3x(acc[i][j], ah[i], al[i], bh[j], blo[j]);
            }
            continue;
        }
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float* a = as + (ks * 8 + t) * LDS_M + i * 16 + g;
                af[i][0] = to_tf32(a[0]);
                af[i][1] = to_tf32(a[8]);
                af[i][2] = to_tf32(a[4 * LDS_M]);
                af[i][3] = to_tf32(a[4 * LDS_M + 8]);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float* b = bs + (ks * 8 + t) * LDS_M + j * 8 + g;
                bf[j][0] = to_tf32(b[0]);
                bf[j][1] = to_tf32(b[4 * LDS_M]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_tf32(acc[i][j], af[i], bf[j]);
        }
    }
    cp_async_wait<0>();

    float* const dwz = DET ? dw + (int64_t)blockIdx.z * p.Ko * p.Ncol : dw;
    if (p.img_pix > 0) {
        const int img = (int)(pix0 / p.img_pix);
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int n = n0 + wn * 32 + j * 8 + 2 * t + u;
                const bool nok = n < p.Ncol;
                const int c = nok ? n % p.C : 0;
                const float sc = nok ? __ldg(p.mod_s + (int64_t)img * p.C + c) : 0.f;
                float dsum = 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int o = o0 + wm * 64 + i * 16 + g + h * 8;
                        if (o >= p.Ko || !nok) continue;
                        const float v = acc[i][j][h * 2 + u];
                        dsum += v * __ldg(p.mod_w + (int64_t)o * p.Ncol + n);
                        drain_add<DET>(dwz + (int64_t)o * p.Ncol + n, v * sc);
                    }
                // the 8 lanes of a column (g = 0..7) share n: reduce before the atomic
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 4);
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 8);
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 16);
                if constexpr (DET) {
                    const int64_t spi = p.img_pix / p.chunk;
                    if (g == 0 && nok)
                        p.mod_ds[wgrad_ds_slot(2 * blockIdx.x + wm, blockIdx.z - img * spi, spi, n / p.C, p.Ncol / p.C) *
                                     ((int64_t)p.N * p.C) + (int64_t)img * p.C + c] = dsum;
                } else {
                    if (g == 0 && nok) atomicAdd(p.mod_ds + (int64_t)img * p.C + c, dsum);
                }
            }
        return;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int o = o0 + wm * 64 + i * 16 + g + h * 8;
            if (o >= p.Ko) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    int n = n0 + wn * 32 + j * 8 + 2 * t + u;
                    if (n < p.Ncol) drain_add<DET>(dwz + (int64_t)o * p.Ncol + n, acc[i][j][h * 2 + u]);
                }
        }
}

// ------------------------------------------------------------------------------------------------
// K splits of the gather GEMM: small-M, deep-K problems (linears) split K so more than a handful of SMs work on them
static unsigned gather_ksplits(const GatherParams& p, const EpiParams& e, int BN) {
    const int64_t tiles = ((p.M + BM - 1) / BM) * ((p.Ncol + BN - 1) / BN);
    const int kblocks = (p.K + BK - 1) / BK;
    const bool plain = !e.bias && !e.noise && !e.residual && e.act == 1 && e.gain == 1.f;
    if (!(plain && tiles <= 16 && kblocks >= 16)) return 1;
    unsigned z = (unsigned)(kblocks / 4);
    if (z > 32) z = 32;
    return z > 1 ? z : 1;
}

// det_ws non-null (the deterministic twin): the split-K partials go to det_ws and det_reduce sums them in split order,
// rounding to TF32 on the way when the epilogue asks for it (no memset, no atomics, no separate rounding pass)
template <int BN, bool VEC, bool SPLIT, bool DET = false>
static int launch_gather(const float* src, const float* wmat, float* out, const GatherParams& p, const EpiParams& e,
                         cudaStream_t st, const float* wlo, float* det_ws = nullptr) {
    size_t smem = (size_t)STAGES * (BM + (SPLIT ? 2 : 1) * BN) * LDS_K * sizeof(float);
    static bool attr_done = false;   // benign race: idempotent
    if (!attr_done) {
        SAE_CUDA_TRY(cudaFuncSetAttribute(conv_gather_kernel<BN, VEC, SPLIT, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    dim3 grid((unsigned)((p.M + BM - 1) / BM), (unsigned)((p.Ncol + BN - 1) / BN));
    grid.z = gather_ksplits(p, e, BN);
    if constexpr (DET) {
        conv_gather_kernel<BN, VEC, SPLIT, true><<<grid, NTHREADS, smem, st>>>(src, wmat, grid.z > 1 ? det_ws : out, p, e, wlo);
        int rc = check_launch("conv_gather_det");
        if (rc == SAE_OK && grid.z > 1) rc = det_reduce(out, det_ws, grid.z, p.M * p.Ncol, false, e.round_tf32, st);
        return rc;
    }
    if (grid.z > 1) SAE_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)p.M * p.Ncol * sizeof(float), st));
    conv_gather_kernel<BN, VEC, SPLIT, false><<<grid, NTHREADS, smem, st>>>(src, wmat, out, p, e, wlo);
    int rc = check_launch("conv_gather");
    // the split-K CTAs add raw partial sums into out: round the finished sums once they are all in
    if (rc == SAE_OK && grid.z > 1 && e.round_tf32) rc = sae_round_tf32(out, out, p.M * p.Ncol, st);
    return rc;
}

template <bool SPLIT, bool DET = false>
static int gather_dispatch_t(const float* src, const float* wmat, float* out, const GatherParams& p, const EpiParams& e,
                             cudaStream_t st, const float* wlo, float* det_ws = nullptr) {
    const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(wmat) | reinterpret_cast<uintptr_t>(wlo)) & 15) == 0;
    const bool vec = (p.Cs % 4 == 0) && aligned;
    if (p.Ncol > 64)
        return vec ? launch_gather<128, true, SPLIT, DET>(src, wmat, out, p, e, st, wlo, det_ws) : launch_gather<128, false, SPLIT, DET>(src, wmat, out, p, e, st, wlo, det_ws);
    if (p.Ncol > 32)
        return vec ? launch_gather<64, true, SPLIT, DET>(src, wmat, out, p, e, st, wlo, det_ws) : launch_gather<64, false, SPLIT, DET>(src, wmat, out, p, e, st, wlo, det_ws);
    return vec ? launch_gather<32, true, SPLIT, DET>(src, wmat, out, p, e, st, wlo, det_ws) : launch_gather<32, false, SPLIT, DET>(src, wmat, out, p, e, st, wlo, det_ws);
}

int conv_gather_dispatch(const float* src, const float* wmat, float* out, const GatherParams& p, const EpiParams& e,
                         cudaStream_t st, const float* wlo) {
    if (p.M == 0 || p.Ncol == 0) return SAE_OK;
    return wlo ? gather_dispatch_t<true>(src, wmat, out, p, e, st, wlo) : gather_dispatch_t<false>(src, wmat, out, p, e, st, nullptr);
}

int conv_gather_dispatch_det(const float* src, const float* wmat, float* out, const GatherParams& p, const EpiParams& e,
                             cudaStream_t st, const float* wlo, void* ws, int64_t* ws_bytes, const char* who) {
    const int BN = p.Ncol > 64 ? 128 : p.Ncol > 32 ? 64 : 32;
    const unsigned z = (p.M == 0 || p.Ncol == 0) ? 1 : gather_ksplits(p, e, BN);
    bool query;
    int rc = det_workspace(ws, ws_bytes, z > 1 ? det_region((int64_t)z * p.M * p.Ncol) : 0, who, &query);
    if (rc || query || p.M == 0 || p.Ncol == 0) return rc;
    float* w = static_cast<float*>(ws);
    return wlo ? gather_dispatch_t<true, true>(src, wmat, out, p, e, st, wlo, w) : gather_dispatch_t<false, true>(src, wmat, out, p, e, st, nullptr, w);
}

template <bool VA, bool VB, bool SPLIT, bool DET>
static int launch_wgrad(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st) {
    size_t smem = (size_t)STAGES * 2 * BK * LDS_M * sizeof(float);
    static bool attr_done = false;
    if (!attr_done) {
        SAE_CUDA_TRY(cudaFuncSetAttribute(conv_wgrad_kernel<VA, VB, SPLIT, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    dim3 grid((unsigned)((p.Ko + 127) / 128), (unsigned)((p.Ncol + 127) / 128), splits);
    conv_wgrad_kernel<VA, VB, SPLIT, DET><<<grid, NTHREADS, smem, st>>>(dy, x, dw, p);
    return check_launch(DET ? "conv_wgrad_det" : "conv_wgrad");
}

template <bool SPLIT, bool DET>
static int launch_wgrad_any(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st,
                            bool va, bool vb) {
    if (va && vb) return launch_wgrad<true, true, SPLIT, DET>(dy, x, dw, p, splits, st);
    if (va) return launch_wgrad<true, false, SPLIT, DET>(dy, x, dw, p, splits, st);
    if (vb) return launch_wgrad<false, true, SPLIT, DET>(dy, x, dw, p, splits, st);
    return launch_wgrad<false, false, SPLIT, DET>(dy, x, dw, p, splits, st);
}

// det non-null: the deterministic twin.  Its splits are planned for DET_SMS SMs, the wgmma kernels are taken as available
// (the library runs on sm_90a only; a device without TMA makes the launch fail), and det->ws == nullptr only plans.
static int wgrad_impl(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, cudaStream_t st,
                      const float* mod_s, const float* mod_w, float* mod_ds, bool split, DetWs* det = nullptr) {
    WgradParams p;
    p.mod_s = mod_s; p.mod_w = mod_w; p.mod_ds = mod_ds;
    p.img_pix = mod_s ? (int64_t)g->P * g->Q : 0;
    p.N = g->N; p.H = g->H; p.W = g->W; p.C = g->C; p.Ko = g->K; p.R = g->R; p.S = g->S; p.P = g->P; p.Q = g->Q;
    p.stride = g->stride; p.pad_t = g->pad_t; p.pad_l = g->pad_l;
    p.Ncol = g->R * g->S * g->C;
    p.Mpix = (int64_t)g->N * g->P * g->Q;
    if (p.Mpix == 0 || p.Ko == 0 || p.Ncol == 0) return SAE_OK;
    const bool al = ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x)) & 15) == 0;
    const bool wg_ok = impl != 1 && al && wgrad_wg_eligible(g) && (det || tc_available());
    if (wg_ok && !split) return wgrad_wg_launch(dy, x, dw, p, st, det);
    int64_t tiles = (int64_t)((p.Ko + 127) / 128) * ((p.Ncol + 127) / 128);
    const int64_t sms = det ? DET_SMS : sm_count();
    int64_t want = (sms * 2 + tiles - 1) / tiles;      // ~2 CTAs per SM
    int64_t kblocks = (p.Mpix + BK - 1) / BK;
    if (want > kblocks) want = kblocks;
    if (want < 1) want = 1;
    if (want > 2048) want = 2048;
    int64_t kb_per = (kblocks + want - 1) / want;
    if (p.img_pix > 0)
        while ((p.img_pix / BK) % kb_per != 0) --kb_per;      // chunks must not straddle images (img_pix % BK == 0)
    p.chunk = kb_per * BK;
    unsigned splits = (unsigned)((p.Mpix + p.chunk - 1) / p.chunk);
    const bool va = (p.Ko % 4 == 0) && al, vb = (p.C % 4 == 0) && al;
    if (det) {
        det->dw_slots = splits;
        det->ds_slots = p.img_pix > 0 ? wgrad_ds_slots((p.Ko + 127) / 128, wg_ok ? 1 : 2, p.img_pix / p.chunk, p.R * p.S) : 0;
        if (!det->ws) return SAE_OK;
        if (wg_ok) return wgrad_split_launch(dy, x, dw, p, splits, st, det);
        p.mod_ds = det->ws_ds;
        return split ? launch_wgrad_any<true, true>(dy, x, det->ws, p, splits, st, va, vb)
                     : launch_wgrad_any<false, true>(dy, x, det->ws, p, splits, st, va, vb);
    }
    if (wg_ok) return wgrad_split_launch(dy, x, dw, p, splits, st);
    return split ? launch_wgrad_any<true, false>(dy, x, dw, p, splits, st, va, vb) : launch_wgrad_any<false, false>(dy, x, dw, p, splits, st, va, vb);
}

int conv_wgrad(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, cudaStream_t st, bool split) {
    return wgrad_impl(dy, x, dw, g, impl, st, nullptr, nullptr, nullptr, split);
}

// plan (DetWs slot counts -> workspace size), check the workspace, run the deterministic drains, then add the slots into dW
// (and ds) in slot order
static int wgrad_det(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw, float* ds,
                     const sae_conv_geom* g, int impl, cudaStream_t st, bool split, void* ws, int64_t* ws_bytes, const char* who) {
    DetWs det;
    int rc = wgrad_impl(dy, x, dw, g, impl, st, s, w_krsc, ds, split, &det);
    if (rc) return rc;
    const int64_t dw_n = (int64_t)g->K * g->R * g->S * g->C, ds_n = (int64_t)g->N * g->C;
    const int64_t dw_bytes = det.dw_slots > 0 ? det_region(det.dw_slots * dw_n) : 0;
    bool query;
    rc = det_workspace(ws, ws_bytes, dw_bytes + (det.ds_slots > 0 ? det_region(det.ds_slots * ds_n) : 0), who, &query);
    if (rc || query || det.dw_slots == 0) return rc;
    det.ws = static_cast<float*>(ws);
    det.ws_ds = reinterpret_cast<float*>(static_cast<char*>(ws) + dw_bytes);
    rc = wgrad_impl(dy, x, dw, g, impl, st, s, w_krsc, ds, split, &det);
    if (rc == SAE_OK) rc = det_reduce(dw, det.ws, det.dw_slots, dw_n, true, 0, st);
    if (rc == SAE_OK && det.ds_slots > 0) rc = det_reduce(ds, det.ws_ds, det.ds_slots, ds_n, true, 0, st);
    return rc;
}

int conv_wgrad_det(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, cudaStream_t st, bool split,
                   void* ws, int64_t* ws_bytes, const char* who) {
    return wgrad_det(dy, x, nullptr, nullptr, dw, nullptr, g, impl, st, split, ws, ws_bytes, who);
}

bool wgrad_modulated_eligible(const sae_conv_geom* g) {
    // whole 32-pixel chunks inside one image, vector loads of both operands
    return g->stride == 1 && g->Q % 32 == 0 && g->C % 32 == 0 && g->C >= 64 && g->K % 32 == 0 && g->R * g->S <= 49 &&
           (int64_t)g->N * g->P * g->Q >= 256;
}

int conv_wgrad_modulated(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw, float* ds,
                         const sae_conv_geom* g, cudaStream_t st, bool split) {
    if (!wgrad_modulated_eligible(g)) return fail(SAE_E_UNSUPPORTED, "modulated wgrad: needs stride 1, Q %% 32 == 0, C and K %% 32 == 0");
    if (((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x)) & 15) != 0)
        return fail(SAE_E_INVALID, "modulated wgrad: pointers must be 16-byte aligned");
    return wgrad_impl(dy, x, dw, g, 0, st, s, w_krsc, ds, split);
}

int conv_wgrad_modulated_det(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw, float* ds,
                             const sae_conv_geom* g, cudaStream_t st, bool split, void* ws, int64_t* ws_bytes, const char* who) {
    if (!wgrad_modulated_eligible(g)) return fail(SAE_E_UNSUPPORTED, "modulated wgrad: needs stride 1, Q %% 32 == 0, C and K %% 32 == 0");
    if (((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x)) & 15) != 0)
        return fail(SAE_E_INVALID, "modulated wgrad: pointers must be 16-byte aligned");
    return wgrad_det(dy, x, s, w_krsc, dw, ds, g, 0, st, split, ws, ws_bytes, who);
}

}  // namespace sae
