// Weight gradient of the convolution on the Hopper tensor cores (wgmma, tf32 inputs, fp32 accumulators in registers).
//
//   dW[o, (tap, c)] += sum_{pixels (n,p,q)}  dy[n,p,q,o] * x[n, p*st - pad_t + r, q*st - pad_l + s, c]
//
// GEMM view: M = out channels (128 per CTA), N = (tap, in channel) columns (128 per CTA), K = output pixels.
//
// TF32 kernel (wgrad_wg_kernel): the reduction walks boxes of 32 output pixels (tw x th x tn, the forward kernel's tiling).
//   * TMA for both operands: per stage one 4-D box of dy per 32-channel block of the M tile, and one 4-D box of x per
//     32-column group of the N tile (a (tap, 32-channel block) pair, read at the box shifted by the tap with element
//     stride = conv stride).  Out-of-image taps and ragged box edges are zero-filled by the TMA unit: no index arithmetic
//     per pixel anywhere.  Both land as [32 pixels][32 channels] in the 128-byte swizzle.
//   * In NHWC both operands are MN-major, and wgmma reads tf32 operands from shared memory K-major only.  So dy goes to wgmma
//     as the register A operand (loaded straight from its tile), and x is transposed into a K-major B tile [128 columns][32
//     pixels] by a dedicated transpose warpgroup.
//   * warps 0..7 = two consumer warpgroups (rows [0, 64) and [64, 128)), warps 8..11 = transposers, warp 12 = TMA producer.
//     A STAGES-deep ring of (dy, x, B) tiles with three mbarriers per stage: full (TMA landed), ready (B transposed),
//     empty (the wgmma group that read the stage has retired: wgmma.wait_group 1 keeps the next group in flight, and the
//     next stage's A fragments load while it runs).
//   * grid = (out-channel tiles, column tiles, pixel splits); partial tiles are reduced into dW with fp32 atomics (dW is
//     zero-initialised by the caller).  Style-modulated mode (img_boxes > 0): boxes hold one image (tn = 1), chunks never
//     straddle images and the drain forms dW += s[n, c] G_n and ds[n, c] += sum_{o, tap} W[o, tap, c] G_n from the unscaled
//     input (ds summed over the CTA's 128 rows in shared memory, one atomic per column).
// Operands are rounded to TF32 (cvt.rna) on their way into the A fragments / the transposed tile, as in the mma.sync kernel.
//
// Split-TF32 kernel (wgrad_split_kernel, the fp32 precision mode): every operand is split into hi = rna_tf32(v),
// lo = rna_tf32(v - hi); both tiles arrive by cp.async (x gathered per pixel), the dy fragments are split in registers, the
// gathered x is transposed into a hi and a lo K-major tile, and each k8 step issues dy_lo x_hi + dy_hi x_lo + dy_hi x_hi.  The
// tensor core's accumulation rounds toward zero, so these wgmma accumulate one stage into partial sums (scale-d = 0 on the
// first) that are added into the accumulators with round-to-nearest fp32 adds.  Its second accumulator set and split
// fragments leave no registers for the pipelined kernel's double-buffered A fragments, so it keeps the two-stage cp.async
// structure.
#include "tc_common.cuh"

namespace sae {

// ================================================================================================ TF32: TMA-fed pipeline
constexpr int WGP_STAGES = 4;
constexpr int WGP_TILE = 128 * 32 * 4;                 // 16 KB: 4 x [32 pixels][32 channels] (dy, x) or [128 columns][32 pixels] (B)
constexpr int WGP_STAGE = 3 * WGP_TILE;                // dy, x, B
constexpr int WGP_CONSUMERS = 256, WGP_TRANSPOSERS = 128;
constexpr int WGP_THREADS = WGP_CONSUMERS + WGP_TRANSPOSERS + 32;
constexpr size_t WGP_SMEM = (size_t)WGP_STAGES * WGP_STAGE + 1024 /*alignment slack*/ + 256 /*barriers*/;

struct WgpParams {
    int Ko, C, Ncol, S;
    int stride, pad_t, pad_l;
    int tw, th, tn, tiles_w, tiles_h;
    int64_t boxes;        // pixel boxes of the output grid
    int64_t chunk;        // boxes per blockIdx.z
    int64_t img_boxes;    // modulated: boxes per image (tn == 1); 0 otherwise
    const float* mod_s;
    const float* mod_w;
    float* mod_ds;
};
struct WgpArgs {
    WgpParams p;
    CUtensorMap dy, x;
};

// DET: dw is the workspace of the deterministic mode, one [Ko, Ncol] slab per pixel split (slot = blockIdx.z), and p.mod_ds
// its ds region, ds_slab = N * C floats per slot (the slot map of wgrad_ds_slot); every element of a slot is stored exactly once
template <bool DET>
__global__ void __launch_bounds__(WGP_THREADS, 1)
wgrad_wg_kernel(float* __restrict__ dw, const __grid_constant__ WgpArgs args, const int64_t ds_slab) {
    const WgpParams& p = args.p;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;       // SWIZZLE_128B needs 1024-byte alignment
    uint8_t* smem_gen = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t bar_full = base + WGP_STAGES * WGP_STAGE;
    const uint32_t bar_ready = bar_full + 8 * WGP_STAGES, bar_empty = bar_ready + 8 * WGP_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int o0 = blockIdx.x * 128, n0 = blockIdx.y * 128;
    const int64_t b0 = (int64_t)blockIdx.z * p.chunk;
    const int KB = (int)((b0 + p.chunk < p.boxes ? b0 + p.chunk : p.boxes) - b0);

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&args.dy) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&args.x) : "memory");
        for (int s = 0; s < WGP_STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_ready + 8 * s, WGP_TRANSPOSERS);
            mbar_init(bar_empty + 8 * s, WGP_CONSUMERS / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == (WGP_CONSUMERS + WGP_TRANSPOSERS) / 32) {
        // ===================================================== TMA producer
        if (lane == 0) {
            // the tile's four 32-column groups: (tap (r, s), channel block) -> x box offset; groups past Ncol are not loaded
            int gc[4], gx[4], gy[4];
            uint32_t bytes = 0;
            const int nm = (p.Ko - o0) / 32 < 4 ? (p.Ko - o0) / 32 : 4;   // dy blocks inside Ko (Ko % 32 == 0)
            bytes += (uint32_t)nm * (WGP_TILE / 4);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = n0 + 32 * j;
                const int tap = col / p.C, r = tap / p.S;
                gc[j] = col < p.Ncol ? col - tap * p.C : -1;
                gy[j] = r - p.pad_t;
                gx[j] = tap - r * p.S - p.pad_l;
                if (col < p.Ncol) bytes += WGP_TILE / 4;
            }
            int tq = (int)(b0 % p.tiles_w);
            const int64_t rest = b0 / p.tiles_w;
            int tp = (int)(rest % p.tiles_h), tb = (int)(rest / p.tiles_h);
            for (int kb = 0; kb < KB; ++kb) {
                const int s = kb % WGP_STAGES;
                mbar_wait(bar_empty + 8 * s, ((uint32_t)(kb / WGP_STAGES) & 1u) ^ 1u);
                const uint32_t sdy = base + (uint32_t)s * WGP_STAGE, sx = sdy + WGP_TILE;
                const int q0 = tq * p.tw, p0 = tp * p.th, nb = tb * p.tn;
                mbar_expect_tx(bar_full + 8 * s, bytes);
                for (int mb = 0; mb < nm; ++mb)
                    tma_load_4d(sdy + mb * (WGP_TILE / 4), &args.dy, bar_full + 8 * s, o0 + 32 * mb, q0, p0, nb);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (gc[j] >= 0)
                        tma_load_4d(sx + j * (WGP_TILE / 4), &args.x, bar_full + 8 * s, gc[j], q0 * p.stride + gx[j],
                                    p0 * p.stride + gy[j], nb);
                if (++tq == p.tiles_w) {
                    tq = 0;
                    if (++tp == p.tiles_h) { tp = 0; ++tb; }
                }
            }
        }
        return;
    }

    if (warp >= WGP_CONSUMERS / 32) {
        // ===================================================== transposers: warp j moves column group j, lane = its column c
        // x group j is [32 pixels][32 channels], element (k, c) at word 32 k + 4 ((c / 4) ^ (k & 7)) + c % 4: for a fixed pixel
        // the 32 lanes read 32 distinct banks.  B is [128 columns n][32 pixels], the 16-byte piece k / 4 of row n at piece
        // (k / 4) ^ (n & 7): each quarter-warp of 16-byte stores (8 consecutive n) covers the 8 pieces of a 128-byte row once.
        const int j = warp - WGP_CONSUMERS / 32, c = lane, n = 32 * j + c;
        for (int kb = 0; kb < KB; ++kb) {
            const int s = kb % WGP_STAGES;
            mbar_wait(bar_full + 8 * s, (uint32_t)(kb / WGP_STAGES) & 1u);
            const float* xs = reinterpret_cast<const float*>(smem_gen + (size_t)s * WGP_STAGE + WGP_TILE) + j * 1024 + (c & 3);
            uint8_t* bt = smem_gen + (size_t)s * WGP_STAGE + 2 * WGP_TILE + n * 128;
#pragma unroll
            for (int k4 = 0; k4 < 8; ++k4) {
                float4 v;
                v.x = rna_tf32(xs[(4 * k4 + 0) * 32 + 4 * ((c >> 2) ^ ((4 * k4 + 0) & 7))]);
                v.y = rna_tf32(xs[(4 * k4 + 1) * 32 + 4 * ((c >> 2) ^ ((4 * k4 + 1) & 7))]);
                v.z = rna_tf32(xs[(4 * k4 + 2) * 32 + 4 * ((c >> 2) ^ ((4 * k4 + 2) & 7))]);
                v.w = rna_tf32(xs[(4 * k4 + 3) * 32 + 4 * ((c >> 2) ^ ((4 * k4 + 3) & 7))]);
                *reinterpret_cast<float4*>(bt + ((k4 ^ (n & 7)) << 4)) = v;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> visible to wgmma
            mbar_arrive(bar_ready + 8 * s);
        }
        return;
    }

    // ===================================================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
    // Rows are permuted onto channels so that the A fragments read dy without bank conflicts.  Warp w (0..7) serves dy
    // block w / 2; the fragment row g = lane / 4 (+ 8 for a1 / a3) is channel 4 c4 + g % 4 of that block, with
    // c4 = 2 (w % 2) + 4 (g / 4) (+ 1 for the rows + 8).  A fragment k column t = lane % 4 (+ 4) is pixel 8 ks + t (+ 4), at
    // word 32 (t (+4)) + 4 (c4 ^ (t (+4))) + g % 4 of the block: c4 ^ t = (c4 % 4 ^ t) + 4 (g / 4) takes the 8 values 0..7
    // over (g / 4, t), and g % 4 the 4 words inside the piece, so the warp's 32 loads hit 32 distinct banks.
    const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
    const int c4a = 2 * (warp & 1) + 4 * (g >> 2), c4b = c4a + 1;
    const bool active = o0 + 64 * wg < p.Ko;
    const int off0 = t * 32 + 4 * (c4a ^ t) + (g & 3), off1 = t * 32 + 4 * (c4b ^ t) + (g & 3);
    const int off2 = (t + 4) * 32 + 4 * (c4a ^ (t + 4)) + (g & 3), off3 = (t + 4) * 32 + 4 * (c4b ^ (t + 4)) + (g & 3);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    uint32_t a0[4][4], a1[4][4];                                       // A fragments of even / odd stages
    auto step = [&](int kb, uint32_t (&a)[4][4]) {
        const int s = kb % WGP_STAGES;
        const uint32_t ph = (uint32_t)(kb / WGP_STAGES) & 1u;
        mbar_wait(bar_full + 8 * s, ph);
        mbar_wait(bar_ready + 8 * s, ph);
        const float* dys = reinterpret_cast<const float*>(smem_gen + (size_t)s * WGP_STAGE) + (warp >> 1) * 1024;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            a[ks][0] = __float_as_uint(rna_tf32(dys[ks * 256 + off0]));
            a[ks][1] = __float_as_uint(rna_tf32(dys[ks * 256 + off1]));
            a[ks][2] = __float_as_uint(rna_tf32(dys[ks * 256 + off2]));
            a[ks][3] = __float_as_uint(rna_tf32(dys[ks * 256 + off3]));
        }
        const uint64_t db = make_wgmma_desc_sw128(base + (uint32_t)s * WGP_STAGE + 2 * WGP_TILE);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_tf32_n128_rs(acc, a[ks], db + (uint64_t)(ks * 2));   // +32 bytes along K
        wgmma_commit();
        wgmma_wait<1>();                                               // the group of stage kb - 1 has retired
        if (kb > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ((kb - 1) % WGP_STAGES));
    };
    if (active) {
        // two A-fragment sets: the in-flight group still reads the other one
        int kb = 0;
        for (; kb + 1 < KB; kb += 2) {
            step(kb, a0);
            step(kb + 1, a1);
        }
        if (kb < KB) step(kb, a0);
        wgmma_wait<0>();
    } else {
        // a warpgroup whose 64 rows all lie past Ko (Ko = 32, 64) issues no MMA; it only keeps the ring turning
        for (int kb = 0; kb < KB; ++kb) {
            const int s = kb % WGP_STAGES;
            const uint32_t ph = (uint32_t)(kb / WGP_STAGES) & 1u;
            mbar_wait(bar_full + 8 * s, ph);
            mbar_wait(bar_ready + 8 * s, ph);
            if (kb > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ((kb - 1) % WGP_STAGES));
        }
    }

    // accumulator fragment: rows g (+ 8) of warp w -> channels o0 + 32 (w / 2) + 4 c4a (c4b) + g % 4, columns n0 + 8 j + 2 t + {0, 1}
    const int oa = o0 + 32 * (warp >> 1) + 4 * c4a + (g & 3), ob = oa + 4;
    float* const dwz = DET ? dw + (int64_t)blockIdx.z * p.Ko * p.Ncol : dw;
    if (p.img_boxes > 0) {
        const int img = (int)(b0 / p.img_boxes);
        // ds: each warp's column sums over its 16 rows (shuffles) land in dsp[warp][column]; then one thread per column adds the
        // 8 warps in a fixed order and issues ONE atomic per column and CTA (few, order-stable contributions per ds element)
        asm volatile("bar.sync 1, %0;" ::"n"(WGP_CONSUMERS) : "memory");   // the ring is free: every stage has been consumed
        float* dsp = reinterpret_cast<float*>(smem_gen);                 // [8 warps][128 columns]
#pragma unroll
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
                    const int o = h ? ob : oa;
                    if (o >= p.Ko || !nok) continue;
                    const float v = acc[4 * j + 2 * h + u];
                    dsum += v * __ldg(p.mod_w + (int64_t)o * p.Ncol + n);
                    drain_add<DET>(dwz + (int64_t)o * p.Ncol + n, v * sc);
                }
                // the 8 lanes of a column (g = 0..7) share n
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 4);
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 8);
                dsum += __shfl_xor_sync(0xffffffffu, dsum, 16);
                if (g == 0) dsp[warp * 128 + 8 * j + 2 * t + u] = dsum;
            }
        asm volatile("bar.sync 1, %0;" ::"n"(WGP_CONSUMERS) : "memory");
        const int tid = threadIdx.x;
        if (tid < 128 && n0 + tid < p.Ncol) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += dsp[w * 128 + tid];
            const int n = n0 + tid;
            if constexpr (DET) {
                const int64_t spi = p.img_boxes / p.chunk;
                p.mod_ds[wgrad_ds_slot(blockIdx.x, blockIdx.z - img * spi, spi, n / p.C, p.Ncol / p.C) * ds_slab + (int64_t)img * p.C + n % p.C] = v;
            } else {
                atomicAdd(p.mod_ds + (int64_t)img * p.C + n % p.C, v);
            }
        }
        return;
    }
    if (!active) return;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int n = n0 + 8 * j + 2 * t;
        if (n >= p.Ncol) continue;                                    // Ncol % 32 == 0: n + 1 < Ncol too
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int o = h ? ob : oa;
            if (o >= p.Ko) continue;
            drain_add<DET>(dwz + (int64_t)o * p.Ncol + n, acc[4 * j + 2 * h]);
            drain_add<DET>(dwz + (int64_t)o * p.Ncol + n + 1, acc[4 * j + 2 * h + 1]);
        }
    }
}

bool wgrad_wg_eligible(const sae_conv_geom* g) {
    return g->K % 32 == 0 && g->C % 32 == 0 && (g->stride == 1 || g->stride == 2) && g->pad_t <= 100 && g->pad_l <= 100;
}

int wgrad_wg_launch(const float* dy, const float* x, float* dw, const WgradParams& wp, cudaStream_t st, DetWs* det) {
    WgpArgs a;
    WgpParams& p = a.p;
    p.Ko = wp.Ko; p.C = wp.C; p.Ncol = wp.Ncol; p.S = wp.S;
    p.stride = wp.stride; p.pad_t = wp.pad_t; p.pad_l = wp.pad_l;
    tile_box(wp.P, wp.Q, 32, 32, p.tw, p.th, p.tn);
    p.tiles_w = (wp.Q + p.tw - 1) / p.tw;
    p.tiles_h = (wp.P + p.th - 1) / p.th;
    const int64_t tiles_n = (wp.N + p.tn - 1) / p.tn;
    p.boxes = (int64_t)p.tiles_w * p.tiles_h * tiles_n;
    p.mod_s = wp.mod_s; p.mod_w = wp.mod_w; p.mod_ds = wp.mod_ds;
    p.img_boxes = 0;
    if (wp.img_pix > 0) {
        if (p.tn != 1) return fail(SAE_E_UNSUPPORTED, "modulated wgrad: pixel boxes must hold one image");
        p.img_boxes = (int64_t)p.tiles_w * p.tiles_h;
    }
    // pixel splits: at least two CTAs' worth per SM — the tensor core adds into its accumulators rounding toward zero, so
    // the pixel run of one CTA sets the error, and this keeps it as short as the mma.sync kernel's — then, one CTA per SM,
    // the fewest splits that fill >= 90 % of the last wave; at least 8 boxes (256 pixels) per CTA keep the 16K atomics of
    // a CTA's drain small against its MMA work
    const int64_t tiles = (int64_t)((p.Ko + 127) / 128) * ((p.Ncol + 127) / 128);
    const int64_t sms = det ? DET_SMS : sm_count();
    const int64_t s_max = p.boxes / 8 > 1 ? p.boxes / 8 : 1;
    const int64_t s_min = (2 * sms + tiles - 1) / tiles;
    int64_t splits = s_max;
    for (int64_t s = s_min; s <= s_max; ++s) {
        const int64_t ctas = tiles * s, waves = (ctas + sms - 1) / sms;
        if (ctas >= (waves * sms * 9 + 9) / 10) { splits = s; break; }
    }
    p.chunk = (p.boxes + splits - 1) / splits;
    if (p.img_boxes > 0) {
        if (p.chunk > p.img_boxes) p.chunk = p.img_boxes;
        while (p.img_boxes % p.chunk != 0) --p.chunk;      // chunks must not straddle images
    }
    splits = (p.boxes + p.chunk - 1) / p.chunk;
    if (splits > 65535) return fail(SAE_E_UNSUPPORTED, "wgrad: %lld pixel splits", (long long)splits);
    if (det) {
        det->dw_slots = splits;
        det->ds_slots = p.img_boxes > 0 ? wgrad_ds_slots((p.Ko + 127) / 128, 1, p.img_boxes / p.chunk, wp.R * wp.S) : 0;
        if (!det->ws) return SAE_OK;
        dw = det->ws;
        p.mod_ds = det->ws_ds;
    }
    int rc = encode_act_map(&a.dy, dy, wp.N, wp.P, wp.Q, wp.Ko, p.tw, p.th, p.tn, 1);
    if (rc) return rc;
    rc = encode_act_map(&a.x, x, wp.N, wp.H, wp.W, wp.C, p.tw, p.th, p.tn, wp.stride);
    if (rc) return rc;
    dim3 grid((unsigned)((p.Ko + 127) / 128), (unsigned)((p.Ncol + 127) / 128), (unsigned)splits);
    if (det) {
        static bool attr_det = false;
        if (!attr_det) {
            SAE_CUDA_TRY(cudaFuncSetAttribute(wgrad_wg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WGP_SMEM));
            attr_det = true;
        }
        wgrad_wg_kernel<true><<<grid, WGP_THREADS, WGP_SMEM, st>>>(dw, a, (int64_t)wp.N * wp.C);
        return check_launch("wgrad_wg_det");
    }
    static bool attr_done = false;
    if (!attr_done) {
        SAE_CUDA_TRY(cudaFuncSetAttribute(wgrad_wg_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WGP_SMEM));
        attr_done = true;
    }
    wgrad_wg_kernel<false><<<grid, WGP_THREADS, WGP_SMEM, st>>>(dw, a, 0);
    return check_launch("wgrad_wg");
}

// ================================================================================================ split-TF32
constexpr int WGR_THREADS = 256;                  // two warpgroups: output-channel rows [0, 64) and [64, 128)
constexpr int WGR_BK = 32;                        // pixels per stage
constexpr int WGR_LD = 128 + 8;                   // row stride (floats) of the pixel-major staging tiles
constexpr int WGR_TILE = WGR_BK * WGR_LD * 4;     // bytes of one pixel-major tile
constexpr int WGR_BT = 128 * WGR_BK * 4;          // the K-major swizzled B tile: 128 rows x 128 bytes = 16 KB
constexpr size_t WGR_SMEM = 2 * (size_t)WGR_BT + 4 * (size_t)WGR_TILE + 1024;

__device__ __forceinline__ void cp_async16_wg(uint32_t s, const void* gmem, bool pred) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(pred ? 16 : 0));
}

// DET: as wgrad_wg_kernel (dw = the workspace's dW slabs, p.mod_ds its ds region with N * C floats per slot)
template <bool DET>
__global__ void __launch_bounds__(WGR_THREADS, 1)
wgrad_split_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dw, const WgradParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;       // SWIZZLE_128B needs 1024-byte alignment
    uint8_t* smem_gen = smem_raw + (base - smem_u32(smem_raw));
    uint8_t* bt = smem_gen;                                            // K-major B tiles: hi, then lo
    const uint32_t bt_s = base;
    float* tiles = reinterpret_cast<float*>(smem_gen + 2 * WGR_BT);    // [stage][A, B][WGR_BK][WGR_LD]
    const uint32_t tiles_s = base + 2 * WGR_BT;

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
    float part[64];                                                    // the current stage's sums
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
        // B: pixel-major [32][136] -> K-major swizzled [128 rows][32 pixels], hi and lo tiles: every thread moves 16-byte pieces
        // (4 pixels of one column), consecutive lanes take consecutive columns, so the reads and the swizzled writes are
        // free of bank conflicts
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) {
            const int idx = tid + WGR_THREADS * qd;
            const int n = idx & 127, c4 = idx >> 7;                    // column n, pixels 4 c4 .. 4 c4 + 3
            uint32_t h[4], l[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) split_tf32(bsrc[(4 * c4 + u) * WGR_LD + n], h[u], l[u]);
            const int off = n * 128 + ((c4 ^ (n & 7)) << 4);
            *reinterpret_cast<uint4*>(bt + off) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4*>(bt + WGR_BT + off) = make_uint4(l[0], l[1], l[2], l[3]);
        }
        // A: m16 x k8 fragments of dy^T (rows = out channels, columns = pixels) from the pixel-major tile (row stride 136
        // floats: conflict-free)
        uint32_t ahi[4][4], alo[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const float* ap = at + (ks * 8 + t) * WGR_LD + r0;
            split_tf32(ap[0], ahi[ks][0], alo[ks][0]);
            split_tf32(ap[8], ahi[ks][1], alo[ks][1]);
            split_tf32(ap[4 * WGR_LD], ahi[ks][2], alo[ks][2]);
            split_tf32(ap[4 * WGR_LD + 8], ahi[ks][3], alo[ks][3]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> visible to wgmma
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
    }

    // accumulator fragment: rows o0 + r0 (+ 8), columns n0 + 8 j + 2 t + {0, 1}
    const int orow = o0 + r0;
    float* const dwz = DET ? dw + (int64_t)blockIdx.z * p.Ko * p.Ncol : dw;
    if (p.img_pix > 0) {
        const int img = (int)(pix0 / p.img_pix);
        // ds: as in the TF32 kernel, one atomic per column and CTA
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
                    drain_add<DET>(dwz + (int64_t)o * p.Ncol + n, v * sc);
                }
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
            const int n = n0 + tid;
            if constexpr (DET) {
                const int64_t spi = p.img_pix / p.chunk;
                p.mod_ds[wgrad_ds_slot(blockIdx.x, blockIdx.z - img * spi, spi, n / p.C, p.Ncol / p.C) * ((int64_t)p.N * p.C) +
                         (int64_t)img * p.C + n % p.C] = v;
            } else {
                atomicAdd(p.mod_ds + (int64_t)img * p.C + n % p.C, v);
            }
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
            if (n < p.Ncol) drain_add<DET>(dwz + (int64_t)o * p.Ncol + n, acc[4 * j + 2 * h]);
            if (n + 1 < p.Ncol) drain_add<DET>(dwz + (int64_t)o * p.Ncol + n + 1, acc[4 * j + 2 * h + 1]);
        }
    }
}

template <bool DET>
static int wgrad_split_launch_t(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st) {
    static bool attr_done = false;
    if (!attr_done) {
        SAE_CUDA_TRY(cudaFuncSetAttribute(wgrad_split_kernel<DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WGR_SMEM));
        attr_done = true;
    }
    dim3 grid((unsigned)((p.Ko + 127) / 128), (unsigned)((p.Ncol + 127) / 128), splits);
    wgrad_split_kernel<DET><<<grid, WGR_THREADS, WGR_SMEM, st>>>(dy, x, dw, p);
    return check_launch(DET ? "wgrad_split_det" : "wgrad_split");
}

int wgrad_split_launch(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st,
                       const DetWs* det) {
    if (!det) return wgrad_split_launch_t<false>(dy, x, dw, p, splits, st);
    WgradParams q = p;
    q.mod_ds = det->ws_ds;
    return wgrad_split_launch_t<true>(dy, x, det->ws, q, splits, st);
}

}  // namespace sae
