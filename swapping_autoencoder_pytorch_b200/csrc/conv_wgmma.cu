// Implicit-GEMM convolution on the Hopper tensor cores: TMA-fed wgmma (tf32 inputs, fp32 accumulators in registers),
// mbarrier pipeline, fused epilogue, TMA store.  sm_90a.
//
//   y[n,p,q,k] = sum_{tap t} sum_c  src[n, p*st + oy_t, q*st + ox_t, c] * wmat[k, t*C + c]
//
// GEMM view: M = output pixels, N = output channels, K = taps x channels.  One CTA computes a
// 128 (pixels) x BLOCK_N (channels) tile:
//   * the 128 pixels are a (tn x th x tw) box of the NHWC output; for tap t the matching A tile is the SAME box of
//     the input shifted by (oy_t, ox_t), out-of-bounds rows/columns zero-filled by the TMA unit (that is the conv's zero
//     padding), landing in shared memory directly in the K-major 128-byte-swizzled layout wgmma consumes: no im2col
//     buffer, no register staging;
//   * tap groups: taps with the same ox whose oy differ by stride * d read the same input rows d output rows apart, so
//     they share ONE 4-D TMA box of th + span rows (box 32ch x tw x (th + span) x tn, element stride = conv stride) and
//     each tap's A tile starts d * tw rows into it (a 3x3 stride-1 conv loads 3 boxes of th + 2 rows per channel block
//     instead of 9 of th rows).  K runs (group, channel block, tap);
//   * B tile = 32 (k) x BLOCK_N rows of the [Cout, taps*C] filter matrix, 2-D TMA, same swizzle;
//   * warps 0..7 = two consumer warpgroups, each issuing m64 x BLOCK_N x k8 wgmma over its 64 tile rows; warp 8 = TMA
//     producer (one lane);
//   * two mbarrier rings (full/empty): A boxes and B tiles.  A consumer warp releases a B stage once the wgmma group that
//     read it has retired (wgmma.wait_group 1 keeps the next group in flight), and an A box once the group of the last
//     tap reading it has;
//   * epilogue: accumulators -> the swizzled staging layout of the output tensor map (reusing the ring) -> bias / noise /
//     leaky-ReLU / residual / TF32 rounding per 32-channel row piece -> TMA store, which also clips ragged tile edges.
// fprop uses it with taps (r - pad_t, s - pad_l); dgrad with taps (pad_t - r, pad_l - s) over dy and the [C, R*S*K]
// transposed filter, a stride-2 data gradient as its four parity classes batched into one launch.  Operands are consumed
// at TF32 precision (low 13 mantissa bits ignored by the tensor core); producers in this library round-to-nearest to TF32
// so that this truncation is exact.  The split-TF32 instantiations (SPLIT = true, the fp32 precision mode) take the filter
// as a (hi, lo) pair of matrices, split the activation tile in registers and issue three register-A wgmma per k8 step.
#include "tc_common.cuh"
#include <mutex>

namespace sae {

// ------------------------------------------------------------------------------------------------ host: driver API
EncodeTiledFn g_encode = nullptr;
static bool g_tc_ok = false;

static void tc_init_once() {
    static std::once_flag once;
    std::call_once(once, [] {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return;
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return;
        if (prop.major != 9) return;
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess) return;
        if (qres != cudaDriverEntryPointSuccess || fn == nullptr) return;
        g_encode = (EncodeTiledFn)fn;
        const char* off = getenv("SAE_DISABLE_TCGEN05");
        g_tc_ok = !(off && off[0] == '1');
    });
}

bool tc_available() {
    tc_init_once();
    return g_tc_ok;
}

// ------------------------------------------------------------------------------------------------ kernel
constexpr int TC_MAX_TAPS = 16;
constexpr int TC_THREADS = 288;                // 2 consumer warpgroups + 1 producer warp
constexpr int TC_CONSUMERS = 256;
constexpr int TC_BK = 32;                      // fp32 elements per K block = one 128-byte swizzle row
constexpr int TC_A_BYTES = 128 * TC_BK * 4;    // 16 KB
constexpr int TC_BOX_PIXELS = 160;             // largest A box (th + span rows of tw pixels): 20 KB

struct TcParams {
    int num_cblk;                 // source channels / 32
    int ntaps;
    int stride;
    int tw, th, tn;               // output tile box (tw*th*tn == 128)
    int tiles_w, tiles_h, tiles_n;
    int ON, OH, OW, Ncol;         // output [ON, OH, OW, Ncol]
    int src_c;                    // source channels
    int o_mul, o_offy, o_offx;    // output sub-grid -> full-resolution pixel (strided outputs of transposed conv)
    int FH, FW;                   // full-resolution output extent (for noise / residual addressing)
    int ngroups;                  // tap groups (tc_plan_groups)
    int box_rows;                 // output rows per A box: th + the largest group span
    short gy[TC_MAX_TAPS], gx[TC_MAX_TAPS];   // group g's box: source pixel = stride * output pixel + (gy, gx)
    unsigned char g_end[TC_MAX_TAPS];         // group g holds taps [g_end[g - 1], g_end[g]) (taps in K order)
    unsigned char a_row[TC_MAX_TAPS];         // first row of the tap's 128-row A tile inside its group's box (d * tw)
    int wk[TC_MAX_TAPS];          // K offset of the tap's filter slice inside a wmat row
    int w_nstride;                // filter rows between consecutive images (0 = one filter for the batch; Ncol = per-sample
                                  // filters [N, Ncol, Ktot], the style-modulated convolution, with tn == 1)
    EpiParams epi;
};

// ------------------------------------------------------------------------------------------------ epilogue pieces
// One 32-column chunk of one accumulator row (= one output pixel): bias / NoiseInjection / leaky-ReLU / gain / residual merge /
// TF32 rounding on 32 values, in the chunk's staging tile ([128 rows][128 bytes], 16-byte pieces XOR-swizzled by (row & 7):
// the layout the SWIZZLE_128B output tensor map reads).
__device__ __forceinline__ void tc_epilogue_math(float (&v)[32], const EpiParams& e, int colb, int64_t pixel, int ncol, bool valid, float nz) {
    uint32_t pos = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        float t = v[j];
        if (e.bias) t += __ldg(e.bias + colb + j);
        t += nz;
        pos |= (t > 0.f ? 1u : 0u) << j;
        if (e.act == 3) t = t > 0.f ? t : t * e.alpha;
        t *= e.gain;
        v[j] = t;
    }
    // activation bit mask: the thread holds the 32 consecutive channels of one pixel = exactly one word.  The backward passes
    // then read 1 bit instead of 32 per element to learn the leaky-ReLU branch (sae_bias_act_backward, sae_fir_act_backward)
    if (e.act_mask && valid) e.act_mask[(pixel * ncol + colb) >> 5] = pos;
    if (e.residual && valid) {
        const float4* r4 = reinterpret_cast<const float4*>(e.residual + pixel * ncol + colb);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float4 r = __ldg(r4 + j);
            v[4 * j + 0] = (v[4 * j + 0] + r.x) * e.res_scale;
            v[4 * j + 1] = (v[4 * j + 1] + r.y) * e.res_scale;
            v[4 * j + 2] = (v[4 * j + 2] + r.z) * e.res_scale;
            v[4 * j + 3] = (v[4 * j + 3] + r.w) * e.res_scale;
        }
    }
    if (e.round_tf32) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = rna_tf32(v[j]);
    }
}

// TF32: <= 96 KB of ring per CTA: two CTAs co-reside on an SM, one runs its epilogue while the other feeds the tensor core.
// Split-TF32 (SPLIT: B_hi and B_lo tiles per stage, a second accumulator set): BLOCK_N = 64 and 32 only (at 128 the
// accumulators, partial sums and split A fragments do not fit the registers without spills), 4 stages; BLOCK_N = 64 takes
// 128 KB and its registers allow one CTA per SM, BLOCK_N = 32 keeps two (96 KB).
template <int BLOCK_N, bool SPLIT>
constexpr int tc_stages() { return SPLIT ? 4 : (BLOCK_N >= 128 ? 3 : 4); }
template <int BLOCK_N, bool SPLIT>
constexpr int tc_min_blocks() { return SPLIT && BLOCK_N >= 64 ? 1 : 2; }

template <int BLOCK_N, bool SPLIT>
constexpr size_t tc_smem_bytes() {
    // A ring (STAGES x 16 KB: STAGES boxes of th rows, or at least two of up to TC_BOX_PIXELS rows) + B ring (STAGES x B, or
    // B_hi + B_lo); the epilogue staging (BLOCK_N/32 chunks of 16 KB) reuses it after the main loop.
    static_assert(tc_stages<BLOCK_N, SPLIT>() * TC_A_BYTES >= 2 * TC_BOX_PIXELS * 128, "the A ring must hold two boxes");
    size_t ring = (size_t)tc_stages<BLOCK_N, SPLIT>() * (TC_A_BYTES + (SPLIT ? 2 : 1) * BLOCK_N * 128);
    size_t epi = (size_t)(BLOCK_N / 32) * TC_A_BYTES;
    return (ring > epi ? ring : epi) + 1024 /*alignment slack*/ + 256 /*barriers*/;
}

// Up to TC_MAX_BATCH problems over the same filter matrix in one launch (the four parity classes of a stride-2 data
// gradient): blockIdx.x walks the problems' tiles back to back.
constexpr int TC_MAX_BATCH = 4;
struct TcBatch {
    int count;
    int tile_end[TC_MAX_BATCH];               // running sum of the problems' pixel-tile counts
    TcParams p[TC_MAX_BATCH];
    CUtensorMap src[TC_MAX_BATCH], out[TC_MAX_BATCH];
    CUtensorMap w;
    CUtensorMap w_lo;                         // split-TF32 only: the low halves of the filter matrix, same geometry as w
};

// SPLIT = false: TF32 operands straight from shared memory (the default).  SPLIT = true: split-TF32, fp32-accurate products:
// w arrives as the pair (hi, lo) = (rna_tf32(w), rna_tf32(w - hi)) in two filter matrices, the activation A is split in
// registers, and every k8 step issues the register-A products A_hi B_hi + A_hi B_lo + A_lo B_hi (A_lo B_lo is below fp32
// rounding and dropped).  The tensor core adds its products into the accumulator rounding toward zero; over thousands of
// k8 steps that bias alone reaches ~1e-5 relative.  So the split path lets wgmma accumulate one stage (32 k) into the partial
// sums `part` (the stage's first wgmma overwrites them: scale-d = 0) and adds `part` into `acc` with round-to-nearest fp32
// adds once per stage.
template <int BLOCK_N, bool SPLIT>
__global__ void __launch_bounds__(TC_THREADS, tc_min_blocks<BLOCK_N, SPLIT>())
conv_wg_kernel(const __grid_constant__ TcBatch batch) {
    int prob = 0;
    while (prob + 1 < batch.count && (int)blockIdx.x >= batch.tile_end[prob]) ++prob;
    const TcParams& p = batch.p[prob];
    const CUtensorMap& map_src = batch.src[prob];
    const CUtensorMap& map_out = batch.out[prob];
    const CUtensorMap& map_w = batch.w;
    constexpr int STAGES = tc_stages<BLOCK_N, SPLIT>();
    constexpr int B_BYTES = BLOCK_N * 128;
    constexpr int B_STAGE = (SPLIT ? 2 : 1) * B_BYTES;
    constexpr int NCHUNK = BLOCK_N / 32;
    constexpr int NACC = BLOCK_N / 2;                                   // fp32 accumulators per thread (m64 x BLOCK_N / 128)

    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;       // SWIZZLE_128B needs 1024-byte alignment
    // A ring [0, A_RING): as many boxes as fit (STAGES of th rows, fewer of th + span rows); B ring: STAGES tiles after it
    constexpr uint32_t A_RING = (uint32_t)STAGES * TC_A_BYTES;
    constexpr uint32_t RING = A_RING + (uint32_t)STAGES * B_STAGE;
    constexpr uint32_t EPI = (uint32_t)NCHUNK * TC_A_BYTES;
    constexpr uint32_t BAR_OFF = RING > EPI ? RING : EPI;
    const uint32_t a_full = base + BAR_OFF;                            // STAGES x 8 bytes each
    const uint32_t a_empty = a_full + 8 * STAGES;
    const uint32_t b_full = a_empty + 8 * STAGES;
    const uint32_t b_empty = b_full + 8 * STAGES;
    uint8_t* smem_gen = smem_raw + (base - smem_u32(smem_raw));       // generic pointer to the aligned base

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // tile coordinates
    int tile = (int)blockIdx.x - (prob > 0 ? batch.tile_end[prob - 1] : 0);
    const int tq = tile % p.tiles_w; tile /= p.tiles_w;
    const int tp = tile % p.tiles_h; tile /= p.tiles_h;
    const int tnb = tile;
    const int q0 = tq * p.tw, p0 = tp * p.th, n0 = tnb * p.tn;
    const int col0 = blockIdx.y * BLOCK_N;
    const uint32_t a_bytes = (uint32_t)(p.box_rows * p.tw * p.tn * 128);   // a multiple of 1024 (tc_plan_groups)
    const int a_slots = (int)(A_RING / a_bytes);                          // >= 2

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_src) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
        if constexpr (SPLIT) asm volatile("prefetch.tensormap [%0];" ::"l"(&batch.w_lo) : "memory");
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(a_full + 8 * s, 1);
            mbar_init(a_empty + 8 * s, TC_CONSUMERS / 32);            // one arrival per consumer warp
            mbar_init(b_full + 8 * s, 1);
            mbar_init(b_empty + 8 * s, TC_CONSUMERS / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == TC_CONSUMERS / 32) {
        // ===================================================== TMA producer: one A box per (group, channel block), one B
        // tile per (channel block, tap), in the consumers' order
        if (lane == 0) {
            const int wrow = col0 + n0 * p.w_nstride;
            int kb = 0, as = 0;
            uint32_t aph = 0;
            for (int g = 0, t0 = 0; g < p.ngroups; t0 = p.g_end[g++]) {
                for (int cb = 0; cb < p.num_cblk; ++cb) {
                    mbar_wait(a_empty + 8 * as, aph ^ 1u);
                    mbar_expect_tx(a_full + 8 * as, a_bytes);
                    tma_load_4d(base + (uint32_t)as * a_bytes, &map_src, a_full + 8 * as, cb * TC_BK, q0 * p.stride + p.gx[g],
                                p0 * p.stride + p.gy[g], n0);
                    if (++as == a_slots) { as = 0; aph ^= 1u; }
                    for (int t = t0; t < p.g_end[g]; ++t, ++kb) {
                        const int s = kb % STAGES;
                        mbar_wait(b_empty + 8 * s, ((uint32_t)(kb / STAGES) & 1u) ^ 1u);
                        const uint32_t sb = base + A_RING + (uint32_t)s * B_STAGE;
                        mbar_expect_tx(b_full + 8 * s, B_STAGE);
                        tma_load_2d(sb, &map_w, b_full + 8 * s, p.wk[t] + cb * TC_BK, wrow);
                        if constexpr (SPLIT) tma_load_2d(sb + B_BYTES, &batch.w_lo, b_full + 8 * s, p.wk[t] + cb * TC_BK, wrow);
                    }
                }
            }
        }
        return;
    }

    // ===================================================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
    const int wg = warp >> 2;
    float acc[NACC];
    float part[SPLIT ? NACC : 1];                                      // split-TF32: the current stage's sums
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    int kb = 0, as = 0, a_done = -1;                                   // a_done: A slot whose last wgmma group is in flight
    uint32_t aph = 0;
    for (int g = 0, t0 = 0; g < p.ngroups; t0 = p.g_end[g++]) {
        for (int cb = 0; cb < p.num_cblk; ++cb) {
            mbar_wait(a_full + 8 * as, aph);
            const uint32_t sbox = base + (uint32_t)as * a_bytes;
            for (int t = t0; t < p.g_end[g]; ++t, ++kb) {
                const int s = kb % STAGES;
                mbar_wait(b_full + 8 * s, (uint32_t)(kb / STAGES) & 1u);
                // the tap's A tile starts a_row rows into the box: a multiple of 8 rows = 1024 bytes, so the swizzle phase
                // (row & 7) and the descriptor's atom alignment are those of the box
                const uint32_t sa = sbox + (uint32_t)p.a_row[t] * 128, sb = base + A_RING + (uint32_t)s * B_STAGE;
                if constexpr (SPLIT) {
                    // A fragments (m16 x k8 per warp, k steps k = 0..3) out of the swizzled tile: rows r = 64 wg + 16 (warp & 3) +
                    // lane / 4 (+ 8), columns 8 k + lane % 4 (+ 4).  r & 7 == lane / 4, so the 16-byte piece (2 k or 2 k + 1) ^ (lane / 4)
                    // and the word lane % 4 put the warp's 32 loads on 32 distinct banks.
                    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
                    const float* arow = reinterpret_cast<const float*>(smem_gen + (sa - base) + (uint32_t)r * 128) + (lane & 3);
                    uint32_t ahi[TC_BK / 8][4], alo[TC_BK / 8][4];
#pragma unroll
                    for (int k = 0; k < TC_BK / 8; ++k) {
                        const int p0 = ((2 * k) ^ (lane >> 2)) * 4, p1 = ((2 * k + 1) ^ (lane >> 2)) * 4;
                        split_tf32(arow[p0], ahi[k][0], alo[k][0]);
                        split_tf32(arow[8 * 32 + p0], ahi[k][1], alo[k][1]);
                        split_tf32(arow[p1], ahi[k][2], alo[k][2]);
                        split_tf32(arow[8 * 32 + p1], ahi[k][3], alo[k][3]);
                    }
                    const uint64_t db = make_wgmma_desc_sw128(sb), dbl = make_wgmma_desc_sw128(sb + B_BYTES);
                    wgmma_fence();
                    Wgmma<BLOCK_N>::template mma_rs<0>(part, alo[0], db);
                    Wgmma<BLOCK_N>::template mma_rs<1>(part, ahi[0], dbl);
                    Wgmma<BLOCK_N>::template mma_rs<1>(part, ahi[0], db);
#pragma unroll
                    for (int k = 1; k < TC_BK / 8; ++k) {
                        Wgmma<BLOCK_N>::template mma_rs<1>(part, alo[k], db + (uint64_t)(k * 2));
                        Wgmma<BLOCK_N>::template mma_rs<1>(part, ahi[k], dbl + (uint64_t)(k * 2));
                        Wgmma<BLOCK_N>::template mma_rs<1>(part, ahi[k], db + (uint64_t)(k * 2));
                    }
                } else {
                    const uint64_t da = make_wgmma_desc_sw128(sa + (uint32_t)wg * (64 * 128)), db = make_wgmma_desc_sw128(sb);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < TC_BK / 8; ++k) {
                        // advance 8 tf32 = 32 bytes along K inside the swizzle atom: +2 in the (addr >> 4) field
                        Wgmma<BLOCK_N>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
                    }
                }
                wgmma_commit();
                if constexpr (SPLIT) {
                    wgmma_wait<0>();       // the next stage's A fragments reuse these registers: retire this group before loading them
                    if (lane == 0) {
                        mbar_arrive(b_empty + 8 * s);
                        if (t + 1 == p.g_end[g]) mbar_arrive(a_empty + 8 * as);
                    }
#pragma unroll
                    for (int i = 0; i < NACC; ++i) acc[i] += part[i];
                } else {
                    wgmma_wait<1>();                                   // the group of B stage kb - 1 has retired
                    if (lane == 0) {
                        if (kb > 0) mbar_arrive(b_empty + 8 * ((kb - 1) % STAGES));
                        if (a_done >= 0) mbar_arrive(a_empty + 8 * a_done);
                    }
                    a_done = -1;
                }
            }
            if constexpr (!SPLIT) a_done = as;                         // released once the group of its last tap retires
            if (++as == a_slots) { as = 0; aph ^= 1u; }
        }
    }
    wgmma_wait<0>();

    // ===================================================== epilogue
    asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory");   // both warpgroups are done reading the ring
    {
        // accumulator fragment (wgmma m64 D layout): warp (warp & 3) of the warpgroup holds rows 16 (warp & 3) + lane / 4
        // (+ 8 for the odd register pair), columns 8 j + 2 (lane & 3) + {0, 1} for j = 0 .. BLOCK_N / 8 - 1
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            const int ch = col >> 5, piece = (col & 31) >> 2;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                uint8_t* dst = smem_gen + (size_t)ch * TC_A_BYTES + (size_t)row * 128 + ((piece ^ (row & 7)) << 4) + (col & 3) * 4;
                *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory");
#pragma unroll 1
    for (int idx = threadIdx.x; idx < 128 * NCHUNK; idx += TC_CONSUMERS) {
        const int row = idx & 127, ch = idx >> 7;
        const int iw = row % p.tw, ih = (row / p.tw) % p.th, in_ = row / (p.tw * p.th);
        const int n = n0 + in_, pp = p0 + ih, qq = q0 + iw;
        const bool valid = n < p.ON && pp < p.OH && qq < p.OW;
        const int64_t pixel = ((int64_t)n * p.FH + pp * p.o_mul + p.o_offy) * p.FW + qq * p.o_mul + p.o_offx;
        float nz = 0.f;
        if (p.epi.noise && valid) nz = __ldg(p.epi.noise_weight) * __ldg(p.epi.noise + pixel);
        uint8_t* stg = smem_gen + (size_t)ch * TC_A_BYTES + (size_t)row * 128;
        float v[32];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 o = *reinterpret_cast<const float4*>(stg + ((j ^ (row & 7)) << 4));
            v[4 * j] = o.x; v[4 * j + 1] = o.y; v[4 * j + 2] = o.z; v[4 * j + 3] = o.w;
        }
        tc_epilogue_math(v, p.epi, col0 + ch * 32, pixel, p.Ncol, valid, nz);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(stg + ((j ^ (row & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // generic-proxy writes -> visible to the TMA store
    asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory");
    if (threadIdx.x == 0) {
        for (int ch = 0; ch < NCHUNK; ++ch) tma_store_4d(&map_out, base + (uint32_t)ch * TC_A_BYTES, col0 + ch * 32, q0, p0, n0);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory stays valid until the stores read it
    }
}

// ------------------------------------------------------------------------------------------------ host side
int encode_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swizzle) {
    if (g_encode == nullptr && !tc_available()) return fail(SAE_E_UNSUPPORTED, "cuTensorMapEncodeTiled is not available on this device / driver");
    CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box,
                          estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(SAE_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return SAE_OK;
}

struct TcProblem {
    const float* src; int SN, SH, SW, SC;      // source activation [SN,SH,SW,SC]
    const float* wmat; int Ncol, Ktot;          // filter matrix [Ncol, Ktot = ntaps*SC]
    const float* wmat_lo;                       // split-TF32: the low halves of wmat (same shape); nullptr = TF32 operands
    int w_per_sample;                           // 1: wmat holds one filter matrix per image, [SN, Ncol, Ktot]
    float* out; int OH, OW;                     // output sub-grid [SN, OH, OW, Ncol] ...
    int o_mul, o_offy, o_offx, FH, FW;          // ... placed at (o_mul*p + o_offy, o_mul*q + o_offx) of the full [SN,FH,FW,Ncol]
    int stride, ntaps;
    int oy[TC_MAX_TAPS], ox[TC_MAX_TAPS], wk[TC_MAX_TAPS];
};

static bool tc_shape_ok(int src_c, int ncol, int ntaps, int stride, int ow) {
    if (src_c % 32 != 0 || ncol % 32 != 0) return false;
    if (ntaps < 1 || ntaps > TC_MAX_TAPS) return false;
    if (stride != 1 && stride != 2) return false;
    int tw = pow2_ceil(ow) < 16 ? pow2_ceil(ow) : 16;
    if (tw * stride > 256) return false;
    return true;
}

static int floor_mod(int a, int m) { return ((a % m) + m) % m; }

// Tap groups.  Source pixel = stride * output pixel + (oy, ox), so two taps with the same ox whose oy differ by stride * d
// read the same input box d output rows apart: they share one A box that starts at the group's smallest oy, and tap t's
// 128-row tile starts a_row[t] = d * tw rows into it.  That start must stay on a 1024-byte swizzle atom (8 rows), which holds
// for one-image tiles (tn == 1) of width 8 or 16; any other tile puts every tap in a group of its own, a box of th rows.
// A group spans at most TC_BOX_PIXELS / tw - th rows (a longer column splits).  The tensor map fixes one box height for the
// problem, th + the largest span, so a group of smaller span loads rows it does not read (stride 2: one in th + 1).
// Taps are ordered by (ox, oy mod stride, oy), which makes each group a contiguous run of the K order.
static void tc_plan_groups(const TcProblem& pr, TcParams& p) {
    const int st = pr.stride;
    const int max_span = p.tn == 1 && (p.tw == 8 || p.tw == 16) ? TC_BOX_PIXELS / p.tw - p.th : 0;
    auto before = [&](int a, int b) {
        if (pr.ox[a] != pr.ox[b]) return pr.ox[a] < pr.ox[b];
        const int ma = floor_mod(pr.oy[a], st), mb = floor_mod(pr.oy[b], st);
        return ma != mb ? ma < mb : pr.oy[a] < pr.oy[b];
    };
    int order[TC_MAX_TAPS];
    for (int t = 0; t < pr.ntaps; ++t) {
        int j = t;
        for (; j > 0 && before(t, order[j - 1]); --j) order[j] = order[j - 1];
        order[j] = t;
    }
    int span = 0;
    p.ngroups = 0;
    for (int i = 0; i < pr.ntaps; ++i) {
        const int t = order[i], g = p.ngroups - 1;
        if (g < 0 || pr.ox[t] != p.gx[g] || floor_mod(pr.oy[t] - p.gy[g], st) != 0 || (pr.oy[t] - p.gy[g]) / st > max_span) {
            p.gy[p.ngroups] = (short)pr.oy[t];
            p.gx[p.ngroups] = (short)pr.ox[t];
            ++p.ngroups;
        }
        const int d = (pr.oy[t] - p.gy[p.ngroups - 1]) / st;
        if (d > span) span = d;
        p.a_row[i] = (unsigned char)(d * p.tw);
        p.wk[i] = pr.wk[t];
        p.g_end[p.ngroups - 1] = (unsigned char)(i + 1);
    }
    p.box_rows = p.th + span;
}

static void tc_fill_params(const TcProblem& pr, const EpiParams& e, TcParams& p) {
    p.num_cblk = pr.SC / 32;
    p.ntaps = pr.ntaps;
    p.stride = pr.stride;
    tile_box(pr.OH, pr.OW, 128, 16, p.tw, p.th, p.tn);
    p.tiles_w = (pr.OW + p.tw - 1) / p.tw;
    p.tiles_h = (pr.OH + p.th - 1) / p.th;
    p.tiles_n = (pr.SN + p.tn - 1) / p.tn;
    p.ON = pr.SN; p.OH = pr.OH; p.OW = pr.OW; p.Ncol = pr.Ncol; p.src_c = pr.SC;
    tc_plan_groups(pr, p);
    p.o_mul = pr.o_mul; p.o_offy = pr.o_offy; p.o_offx = pr.o_offx; p.FH = pr.FH; p.FW = pr.FW;
    p.w_nstride = pr.w_per_sample ? pr.Ncol : 0;
    p.epi = e;
}

static int tc_encode_filter(const TcProblem& pr, const float* wmat, int b_rows, CUtensorMap* mw) {
    cuuint64_t dims[2] = {(cuuint64_t)pr.Ktot, (cuuint64_t)pr.Ncol * (cuuint64_t)(pr.w_per_sample ? pr.SN : 1)};
    cuuint64_t strides[1] = {(cuuint64_t)pr.Ktot * 4};
    cuuint32_t box[2] = {32, (cuuint32_t)b_rows};
    cuuint32_t es[2] = {1, 1};
    return encode_map(mw, wmat, 2, dims, strides, box, es);
}

int encode_act_map(CUtensorMap* m, const float* ptr, int N, int H, int W, int C, int tw, int th, int tn, int stride) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
    cuuint32_t box[4] = {32, (cuuint32_t)(tw * stride), (cuuint32_t)(th * stride), (cuuint32_t)tn};
    cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    return encode_map(m, ptr, 4, dims, strides, box, es);
}

static int tc_encode_maps(const TcProblem& pr, const TcParams& p, int b_rows, CUtensorMap* msrc, CUtensorMap* mw, CUtensorMap* mout) {
    {
        int rc = encode_act_map(msrc, pr.src, pr.SN, pr.SH, pr.SW, pr.SC, p.tw, p.box_rows, p.tn, pr.stride);
        if (rc) return rc;
    }
    {
        int rc = tc_encode_filter(pr, pr.wmat, b_rows, mw);
        if (rc) return rc;
    }
    {
        cuuint64_t dims[4] = {(cuuint64_t)pr.Ncol, (cuuint64_t)pr.OW, (cuuint64_t)pr.OH, (cuuint64_t)pr.SN};
        cuuint64_t strides[3] = {(cuuint64_t)pr.o_mul * pr.Ncol * 4, (cuuint64_t)pr.o_mul * pr.FW * pr.Ncol * 4,
                                 (cuuint64_t)pr.FH * pr.FW * pr.Ncol * 4};
        cuuint32_t box[4] = {32, (cuuint32_t)p.tw, (cuuint32_t)p.th, (cuuint32_t)p.tn};
        cuuint32_t es[4] = {1, 1, 1, 1};
        int rc = encode_map(mout, pr.out + ((int64_t)pr.o_offy * pr.FW + pr.o_offx) * pr.Ncol, 4, dims, strides, box, es);
        if (rc) return rc;
    }
    return SAE_OK;
}

// one-tile-per-CTA launch of up to TC_MAX_BATCH problems that share the filter matrix, the column count and the epilogue
template <int BLOCK_N, bool SPLIT>
static int tc_launch_batch(const TcProblem* prs, int count, const EpiParams& e, cudaStream_t st) {
    TcBatch b;
    if (count < 1 || count > TC_MAX_BATCH) return fail(SAE_E_INVALID, "conv_wg: batch of %d problems", count);
    b.count = count;
    int tiles = 0;
    for (int i = 0; i < count; ++i) {
        tc_fill_params(prs[i], e, b.p[i]);
        if (prs[i].w_per_sample && b.p[i].tn != 1) return fail(SAE_E_UNSUPPORTED, "conv_wg: per-sample filters need one image per tile");
        CUtensorMap mw;
        int rc = tc_encode_maps(prs[i], b.p[i], BLOCK_N, &b.src[i], &mw, &b.out[i]);
        if (rc) return rc;
        if (i == 0) b.w = mw;
        else if (prs[i].wmat != prs[0].wmat || prs[i].wmat_lo != prs[0].wmat_lo || prs[i].Ncol != prs[0].Ncol ||
                 prs[i].Ktot != prs[0].Ktot)
            return fail(SAE_E_INVALID, "conv_wg: batched problems must share the filter matrix");
        tiles += b.p[i].tiles_w * b.p[i].tiles_h * b.p[i].tiles_n;
        b.tile_end[i] = tiles;
    }
    if (SPLIT) {
        int rc = tc_encode_filter(prs[0], prs[0].wmat_lo, BLOCK_N, &b.w_lo);
        if (rc) return rc;
    }
    constexpr size_t smem = tc_smem_bytes<BLOCK_N, SPLIT>();
    static bool attr_done = false;
    if (!attr_done) {
        SAE_CUDA_TRY(cudaFuncSetAttribute(conv_wg_kernel<BLOCK_N, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    dim3 grid((unsigned)tiles, (unsigned)(prs[0].Ncol / BLOCK_N));
    conv_wg_kernel<BLOCK_N, SPLIT><<<grid, TC_THREADS, smem, st>>>(b);
    return check_launch("conv_wg");
}

static int tc_dispatch(const TcProblem* prs, int count, const EpiParams& e, cudaStream_t st) {
    const int ncol = prs[0].Ncol;
    if (prs[0].wmat_lo) {
        if (ncol % 64 == 0) return tc_launch_batch<64, true>(prs, count, e, st);
        return tc_launch_batch<32, true>(prs, count, e, st);
    }
    if (ncol % 128 == 0) return tc_launch_batch<128, false>(prs, count, e, st);
    if (ncol % 64 == 0) return tc_launch_batch<64, false>(prs, count, e, st);
    return tc_launch_batch<32, false>(prs, count, e, st);
}

static bool ptr_ok(const void* a, const void* b, const void* c, const void* d = nullptr) {
    return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
             reinterpret_cast<uintptr_t>(d)) & 15) == 0;
}

bool tc_fprop_eligible(const sae_conv_geom* g) {
    if (g->R * g->S > TC_MAX_TAPS) return false;
    if (g->pad_t > 100 || g->pad_l > 100) return false;
    return tc_shape_ok(g->C, g->K, g->R * g->S, g->stride, g->Q);
}

bool tc_dgrad_eligible(const sae_conv_geom* g) {
    if (g->stride != 1 && g->stride != 2) return false;
    if (g->R * g->S > TC_MAX_TAPS) return false;
    if (g->pad_t > 100 || g->pad_l > 100) return false;
    return tc_shape_ok(g->K, g->C, g->R * g->S, 1, (g->W + g->stride - 1) / g->stride);
}

int tc_fprop(const float* x, const float* w, float* y, const sae_conv_geom* g, const EpiParams& e, cudaStream_t st,
             const float* w_lo) {
    if (!ptr_ok(x, w, y, w_lo)) return fail(SAE_E_INVALID, "conv2d_fprop(wgmma): pointers must be 16-byte aligned");
    TcProblem pr;
    pr.w_per_sample = 0;
    pr.wmat_lo = w_lo;
    pr.src = x; pr.SN = g->N; pr.SH = g->H; pr.SW = g->W; pr.SC = g->C;
    pr.wmat = w; pr.Ncol = g->K; pr.Ktot = g->R * g->S * g->C;
    pr.out = y; pr.OH = g->P; pr.OW = g->Q;
    pr.o_mul = 1; pr.o_offy = 0; pr.o_offx = 0; pr.FH = g->P; pr.FW = g->Q;
    pr.stride = g->stride; pr.ntaps = g->R * g->S;
    for (int r = 0; r < g->R; ++r)
        for (int s = 0; s < g->S; ++s) {
            const int t = r * g->S + s;
            pr.oy[t] = r - g->pad_t; pr.ox[t] = s - g->pad_l; pr.wk[t] = t * g->C;
        }
    return tc_dispatch(&pr, 1, e, st);
}

// Per-sample filters (the style-modulated convolution, stylegan2_layers.py:284-323): image n is convolved with filter matrix n.
// Every pixel tile must lie in one image (tn == 1), which holds for stride-1 maps whose height is a multiple of 16 and whose
// width is a multiple of 8; anything else reports UNSUPPORTED and the caller scales the input instead.
bool tc_per_sample_eligible(const sae_conv_geom* g, int dgrad) {
    if (g->stride != 1 || g->R * g->S > TC_MAX_TAPS) return false;
    const int src_c = dgrad ? g->K : g->C, ncol = dgrad ? g->C : g->K;
    const int oh = dgrad ? g->H : g->P, ow = dgrad ? g->W : g->Q;
    if (src_c % 32 != 0 || ncol % 32 != 0 || oh % 16 != 0 || ow % 8 != 0) return false;
    if (g->R > 3 || g->S > 3) return false;
    return (int64_t)g->N * oh * ow >= 2 * 128;
}

int tc_conv_per_sample(const float* src, const float* w, float* out, const sae_conv_geom* g, int dgrad, const EpiParams& e, cudaStream_t st,
                       const float* w_lo) {
    if (!tc_per_sample_eligible(g, dgrad)) return fail(SAE_E_UNSUPPORTED, "per-sample conv: shape outside the per-sample kernel");
    if (!ptr_ok(src, w, out, w_lo)) return fail(SAE_E_INVALID, "per-sample conv: pointers must be 16-byte aligned");
    TcProblem pr;
    pr.w_per_sample = 1;
    pr.wmat_lo = w_lo;
    pr.stride = 1; pr.o_mul = 1; pr.o_offy = 0; pr.o_offx = 0; pr.ntaps = g->R * g->S;
    pr.src = src; pr.wmat = w; pr.out = out; pr.SN = g->N;
    if (!dgrad) {
        pr.SH = g->H; pr.SW = g->W; pr.SC = g->C; pr.Ncol = g->K; pr.Ktot = g->R * g->S * g->C;
        pr.OH = g->P; pr.OW = g->Q; pr.FH = g->P; pr.FW = g->Q;
    } else {
        pr.SH = g->P; pr.SW = g->Q; pr.SC = g->K; pr.Ncol = g->C; pr.Ktot = g->R * g->S * g->K;
        pr.OH = g->H; pr.OW = g->W; pr.FH = g->H; pr.FW = g->W;
    }
    for (int r = 0; r < g->R; ++r)
        for (int s_ = 0; s_ < g->S; ++s_) {
            const int t = r * g->S + s_;
            pr.oy[t] = dgrad ? g->pad_t - r : r - g->pad_t;
            pr.ox[t] = dgrad ? g->pad_l - s_ : s_ - g->pad_l;
            pr.wk[t] = t * pr.SC;
        }
    return tc_dispatch(&pr, 1, e, st);
}

// The pixels of the stride-2 parity classes that no filter tap reaches (bit 2 (y & 1) + (x & 1) of `empty`): the epilogue of
// a zero accumulator, in the order of tc_epilogue_math, and their activation mask words.  One thread per element of dx; with
// C % 32 == 0 (the wgmma path's column granularity) the 32 lanes of a warp are the 32 channels of one pixel = one mask word.
__global__ void __launch_bounds__(256)
tc_dgrad_empty_kernel(float* __restrict__ dx, const EpiParams e, int64_t total, int H, int W, int C, unsigned empty) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pixel = i / C;
        const int col = (int)(i - pixel * C);
        const int x = (int)(pixel % W), y = (int)((pixel / W) % H);
        if (!((empty >> ((y & 1) * 2 + (x & 1))) & 1u)) continue;        // uniform over the warp
        float t = 0.f;
        if (e.bias) t += __ldg(e.bias + col);
        if (e.noise) t += __ldg(e.noise_weight) * __ldg(e.noise + pixel);
        const uint32_t pos = __ballot_sync(0xffffffffu, t > 0.f);
        if (e.act == 3) t = t > 0.f ? t : t * e.alpha;
        t *= e.gain;
        if (e.act_mask && (i & 31) == 0) e.act_mask[i >> 5] = pos;
        if (e.residual) t = (t + __ldg(e.residual + i)) * e.res_scale;
        if (e.round_tf32) t = rna_tf32(t);
        dx[i] = t;
    }
}

int tc_dgrad(const float* dy, const float* wt, float* dx, const sae_conv_geom* g, const EpiParams& e, cudaStream_t st,
             const float* wt_lo) {
    if (!ptr_ok(dy, wt, dx, wt_lo)) return fail(SAE_E_INVALID, "conv2d_dgrad(wgmma): pointers must be 16-byte aligned");
    TcProblem pr;
    pr.w_per_sample = 0;
    pr.wmat_lo = wt_lo;
    pr.src = dy; pr.SN = g->N; pr.SH = g->P; pr.SW = g->Q; pr.SC = g->K;
    pr.wmat = wt; pr.Ncol = g->C; pr.Ktot = g->R * g->S * g->K;
    pr.stride = 1; pr.FH = g->H; pr.FW = g->W;
    const int st_ = g->stride;
    if (st_ == 1) {
        pr.out = dx; pr.OH = g->H; pr.OW = g->W; pr.o_mul = 1; pr.o_offy = 0; pr.o_offx = 0;
        pr.ntaps = g->R * g->S;
        for (int r = 0; r < g->R; ++r)
            for (int s = 0; s < g->S; ++s) {
                const int t = r * g->S + s;
                pr.oy[t] = g->pad_t - r; pr.ox[t] = g->pad_l - s; pr.wk[t] = t * g->K;
            }
        return tc_dispatch(&pr, 1, e, st);
    }
    // stride 2 (the generator's transposed convolution and the data-gradient of the strided convs): the output
    // splits into 4 parity classes (ho, wo); class outputs x[2i+ho, 2j+wo] only see taps with r = (ho + pad_t) mod 2,
    // s = (wo + pad_l) mod 2, read at source offset (ho + pad_t - r) / 2 — four dense stride-1 problems writing
    // interleaved sub-grids (the output tensor map carries the doubled strides), batched into one launch.
    // a class no tap reaches (R == 1 or S == 1) has a zero accumulator: with a trivial epilogue its pixels are 0, otherwise
    // they take the epilogue of 0 and their mask words from tc_dgrad_empty_kernel
    unsigned empty = 0;
    for (int ho = 0; ho < 2; ++ho)
        for (int wo = 0; wo < 2; ++wo) {
            const int rp = (ho + g->pad_t) & 1, sp = (wo + g->pad_l) & 1;
            if (rp >= g->R || sp >= g->S) empty |= 1u << (ho * 2 + wo);
        }
    if (empty) {
        const int64_t total = (int64_t)g->N * g->H * g->W * g->C;
        if (!e.bias && !e.noise && !e.residual && !e.act_mask) {
            SAE_CUDA_TRY(cudaMemsetAsync(dx, 0, (size_t)total * sizeof(float), st));
        } else {
            int64_t blocks = (total + 255) / 256;
            if (blocks > (int64_t)sm_count() * 16) blocks = (int64_t)sm_count() * 16;
            tc_dgrad_empty_kernel<<<(unsigned)blocks, 256, 0, st>>>(dx, e, total, g->H, g->W, g->C, empty);
            int rc = check_launch("conv_wg(dgrad, empty parity classes)");
            if (rc) return rc;
        }
    }
    TcProblem cls_pr[TC_MAX_BATCH];
    int ncls = 0;
    for (int ho = 0; ho < 2; ++ho)
        for (int wo = 0; wo < 2; ++wo) {
            const int rp = (ho + g->pad_t) & 1, sp = (wo + g->pad_l) & 1;
            if (rp >= g->R || sp >= g->S) continue;
            if (ho >= g->H || wo >= g->W) continue;
            pr.out = dx; pr.o_mul = 2; pr.o_offy = ho; pr.o_offx = wo;
            pr.OH = (g->H - ho + 1) / 2; pr.OW = (g->W - wo + 1) / 2;
            int nt = 0;
            for (int r = rp; r < g->R; r += 2)
                for (int s = sp; s < g->S; s += 2) {
                    // exact division: (ho + pad_t - r) is even; C++ division truncates toward zero, so floor by hand
                    const int ny = ho + g->pad_t - r, nx = wo + g->pad_l - s;
                    pr.oy[nt] = ny >= 0 ? ny / 2 : -((-ny) / 2);
                    pr.ox[nt] = nx >= 0 ? nx / 2 : -((-nx) / 2);
                    pr.wk[nt] = (r * g->S + s) * g->K;
                    ++nt;
                }
            pr.ntaps = nt;
            cls_pr[ncls++] = pr;
        }
    if (ncls == 0) return SAE_OK;
    return tc_dispatch(cls_pr, ncls, e, st);
}

}  // namespace sae
