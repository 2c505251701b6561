// Internal declarations shared by api.cu, conv_generic.cu and conv_wgmma.cu.
#pragma once
#include "common.cuh"

namespace sae {

struct GatherParams {
    int N, OH, OW;          // output pixel space, M = N*OH*OW
    int IH, IW, Cs;         // source activation
    int R, S;
    int SY, DY, OFFY, OFFX, DIV;
    int Ncol;               // output channels
    int K;                  // R*S*Cs
    int64_t M;
};

// wgrad: C[o, n=(tap,c)] += sum_{pixel} dy[pixel, o] * x[gather(pixel, tap), c]
struct WgradParams {
    int N, H, W, C;       // x
    int Ko, R, S;         // dy channels / filter
    int P, Q;
    int stride, pad_t, pad_l;
    int Ncol;             // R*S*C
    int64_t Mpix;         // N*P*Q
    int64_t chunk;        // pixels per blockIdx.z (multiple of 32)
    // style-modulated convolution (stylegan2_layers.py:284-323 as "dense conv of x * s with a shared filter W"): x arrives
    // UNSCALED and every chunk lies inside one image n, so the CTA's tile is G_n[o, (tap, c)] = sum_pixels dy x, from which
    // the drain forms both gradients: dW += s[n, c] G_n, ds[n, c] += sum_{o, tap} W[o, tap, c] G_n.
    int64_t img_pix;      // P*Q when modulated, 0 otherwise
    const float* mod_s;   // [N, C]
    const float* mod_w;   // [Ko, R*S*C], the filter the forward pass used
    float* mod_ds;        // [N, C], accumulated
};
// conv_generic.cu
// wlo non-null: split-TF32 operands, the filter given as the pair (wmat, wlo) = (hi, lo)
int conv_gather_dispatch(const float* src, const float* wmat, float* out, const GatherParams& p, const EpiParams& e,
                         cudaStream_t st, const float* wlo = nullptr);
// impl: 0 = the wgmma kernel where the channel counts allow it (wgrad_wgmma.cu), 1 = the mma.sync kernel;
// split: split-TF32 operands (both split in-kernel)
int conv_wgrad(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, cudaStream_t st, bool split = false);
// weight gradient of the style-modulated convolution (per-sample filters W * s[n]) from the unscaled input
bool wgrad_modulated_eligible(const sae_conv_geom* g);
int conv_wgrad_modulated(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw, float* ds,
                         const sae_conv_geom* g, cudaStream_t st, bool split = false);

// conv_wgmma.cu
bool tc_available();
bool tc_fprop_eligible(const sae_conv_geom* g);
bool tc_dgrad_eligible(const sae_conv_geom* g);
// w_lo / wt_lo non-null: split-TF32 operands, the filter given as the pair (w, w_lo) = (hi, lo) (sae_split_tf32)
int tc_fprop(const float* x, const float* w, float* y, const sae_conv_geom* g, const EpiParams& e, cudaStream_t st,
             const float* w_lo = nullptr);
int tc_dgrad(const float* dy, const float* wt, float* dx, const sae_conv_geom* g, const EpiParams& e, cudaStream_t st,
             const float* wt_lo = nullptr);
// wgrad_wgmma.cu: weight gradient (plain and modulated) on wgmma; needs K % 32 == 0, C % 32 == 0, stride 1 or 2, and
// 16-byte aligned dy and x (other shapes take the mma.sync kernel).  wgrad_wg_launch: TF32 operands, TMA-fed pipeline,
// chooses its own pixel splits; wgrad_split_launch: split-TF32 operands, p.chunk pixels per split
bool wgrad_wg_eligible(const sae_conv_geom* g);
int wgrad_wg_launch(const float* dy, const float* x, float* dw, const WgradParams& p, cudaStream_t st);
int wgrad_split_launch(const float* dy, const float* x, float* dw, const WgradParams& p, unsigned splits, cudaStream_t st);
// style-modulated convolution: per-sample filters (forward / data gradient)
bool tc_per_sample_eligible(const sae_conv_geom* g, int dgrad);
int tc_conv_per_sample(const float* src, const float* w, float* out, const sae_conv_geom* g, int dgrad, const EpiParams& e,
                       cudaStream_t st, const float* w_lo = nullptr);

}  // namespace sae
