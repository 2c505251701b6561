// Adaptive discriminator augmentation (INTEGRATION §2h): StyleGAN2-ADA's geometric and colour transforms ('bgc') of the
// images D sees, with the augmentation probability p tuned on the device.
//   * sae_augment_params: every image's G_inv (3x3) and C (4x4) from its draws and the device p;
//   * sae_augment_sample: reflect pad + sym6 2x upsample (computed on the fly) + bilinear sample on the transformed grid;
//   * sae_augment_sample_adjoint: its adjoint in gather form, one thread per input pixel;
//   * sae_augment_color / _adjoint: the per-pixel colour matrix (with the identity-copy select) and its transpose;
//   * sae_ada_adjust: p += sign(E[sign(D(real))] - target) * step, clamped at 0.
// No float atomics anywhere: every output element is written by one thread, so the results are bitwise reproducible.
#include <cmath>

#include "common.cuh"

namespace sae {

// 2 * sym6 / sum(sym6) = sqrt(2) * sym6: one axis of the upsampling filter with gain 4 (2 per axis), normalised to sum 2
#define SAE_SYM6_G(v) ((float)((v) * 1.4142135623730951))
__constant__ float c_aug_g[12] = {
    SAE_SYM6_G(0.015404109327027373), SAE_SYM6_G(0.0034907120842174702), SAE_SYM6_G(-0.11799011114819057),
    SAE_SYM6_G(-0.048311742585633), SAE_SYM6_G(0.4910559419267466), SAE_SYM6_G(0.787641141030194),
    SAE_SYM6_G(0.3379294217276218), SAE_SYM6_G(-0.07263752278646252), SAE_SYM6_G(-0.021060292512300564),
    SAE_SYM6_G(0.04472490177066578), SAE_SYM6_G(0.0017677118642428036), SAE_SYM6_G(-0.007800708325034148)};
#undef SAE_SYM6_G

constexpr int AUG_HZ = 3;            // Hz_pad: the sample grid is 2 (H + 2 Hz_pad) x 2 (W + 2 Hz_pad)

// ------------------------------------------------------------------------------------------------- matrices from draws
struct M3 { double m[3][3]; };
struct M4 { double m[4][4]; };

__device__ __forceinline__ M3 m3_eye() { M3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = i == j; return r; }
__device__ __forceinline__ M4 m4_eye() { M4 r; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.m[i][j] = i == j; return r; }

__device__ __forceinline__ M3 m3_mul(const M3& a, const M3& b) {
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
    return r;
}

__device__ __forceinline__ M4 m4_mul(const M4& a, const M4& b) {
    M4 r;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j] + a.m[i][3] * b.m[3][j];
    return r;
}

__device__ __forceinline__ M3 scale2d(double sx, double sy) { M3 r = m3_eye(); r.m[0][0] = sx; r.m[1][1] = sy; return r; }
__device__ __forceinline__ M3 translate2d(double tx, double ty) { M3 r = m3_eye(); r.m[0][2] = tx; r.m[1][2] = ty; return r; }
__device__ __forceinline__ M3 rotate2d(double t) {
    M3 r = m3_eye();
    const double c = cos(t), s = sin(t);
    r.m[0][0] = c; r.m[0][1] = -s; r.m[1][0] = s; r.m[1][1] = c;
    return r;
}

// One thread per image.  Column layout of the draws (fixed; tests/ada_oracle.py restates it):
//   u[n, 0..20]: 0 x-flip gate, 1 x-flip, 2 rot90 gate, 3 rot90, 4 int-translation gate, 5 / 6 its x / y, 7 iso-scale gate,
//     8 pre-rotation gate, 9 pre-rotation, 10 aniso gate, 11 post-rotation gate, 12 post-rotation, 13 frac-translation gate,
//     14 brightness gate, 15 contrast gate, 16 luma-flip gate, 17 luma flip, 18 hue gate, 19 hue, 20 saturation gate;
//   z[n, 0..6]: 0 iso scale, 1 aniso scale, 2 / 3 frac translation x / y, 4 brightness, 5 contrast, 6 saturation.
__global__ void aug_params_kernel(const float* __restrict__ u, const float* __restrict__ z, const float* __restrict__ p_dev,
                                  float* __restrict__ rec, int N, int H, int W) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float* un = u + (int64_t)n * SAE_AUG_UNIFORMS;
    const float* zn = z + (int64_t)n * SAE_AUG_NORMALS;
    const double p = (double)*p_dev;
    const double p_rot = 1.0 - sqrt(fmin(fmax(1.0 - p, 0.0), 1.0));
    const double pi = 3.14159265358979323846;
    auto U = [&](int k) { return (double)__ldg(un + k); };
    auto Z = [&](int k) { return (double)__ldg(zn + k); };
    // G_inv = I * f1^-1 * f2^-1 * ... (right-multiplied); every inverse is written out in closed form
    M3 G = m3_eye();
    if (U(0) < p) G = m3_mul(G, scale2d(1.0 - 2.0 * floor(2.0 * U(1)), 1.0));
    if (U(2) < p) G = m3_mul(G, rotate2d(pi / 2 * floor(4.0 * U(3))));
    if (U(4) < p) G = m3_mul(G, translate2d(-rint((2.0 * U(5) - 1.0) * 0.125 * W), -rint((2.0 * U(6) - 1.0) * 0.125 * H)));
    if (U(7) < p) { const double s = exp2(0.2 * Z(0)); G = m3_mul(G, scale2d(1.0 / s, 1.0 / s)); }
    if (U(8) < p_rot) G = m3_mul(G, rotate2d((2.0 * U(9) - 1.0) * pi));
    if (U(10) < p) { const double s = exp2(0.2 * Z(1)); G = m3_mul(G, scale2d(1.0 / s, s)); }
    if (U(11) < p_rot) G = m3_mul(G, rotate2d((2.0 * U(12) - 1.0) * pi));
    if (U(13) < p) G = m3_mul(G, translate2d(-0.125 * Z(2) * W, -0.125 * Z(3) * H));
    // C = f5 * f4 * ... * f1 * I (left-multiplied)
    const double v = 1.0 / sqrt(3.0);
    M4 C = m4_eye();
    if (U(14) < p) { M4 f = m4_eye(); const double b = 0.2 * Z(4); f.m[0][3] = f.m[1][3] = f.m[2][3] = b; C = m4_mul(f, C); }
    if (U(15) < p) { M4 f = m4_eye(); const double c = exp2(0.5 * Z(5)); f.m[0][0] = f.m[1][1] = f.m[2][2] = c; C = m4_mul(f, C); }
    if (U(16) < p) {
        const double i = floor(2.0 * U(17));
        M4 f = m4_eye();
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) f.m[a][b] -= 2.0 * v * v * i;
        C = m4_mul(f, C);
    }
    if (U(18) < p) {
        const double t = (2.0 * U(19) - 1.0) * pi, c = cos(t), s = sin(t), cc = 1.0 - c;
        M4 f = m4_eye();
        // Rodrigues about the unit luma axis (v, v, v)
        f.m[0][0] = v * v * cc + c;     f.m[0][1] = v * v * cc - v * s; f.m[0][2] = v * v * cc + v * s;
        f.m[1][0] = v * v * cc + v * s; f.m[1][1] = v * v * cc + c;     f.m[1][2] = v * v * cc - v * s;
        f.m[2][0] = v * v * cc - v * s; f.m[2][1] = v * v * cc + v * s; f.m[2][2] = v * v * cc + c;
        C = m4_mul(f, C);
    }
    if (U(20) < p) {
        const double s = exp2(Z(6));
        M4 f;
        for (int a = 0; a < 4; ++a)
            for (int b = 0; b < 4; ++b) {
                const double vv = (a < 3 && b < 3) ? v * v : 0.0;
                f.m[a][b] = vv + ((a == b ? 1.0 : 0.0) - vv) * s;
            }
        C = m4_mul(f, C);
    }
    float* r = rec + (int64_t)n * SAE_AUG_RECORD;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[3 * i + j] = (float)G.m[i][j];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) r[9 + 4 * i + j] = (float)C.m[i][j];
    for (int k = 25; k < SAE_AUG_RECORD; ++k) r[k] = 0.f;
}

// ------------------------------------------------------------------------------------------------- geometric resampler
struct AugGeom {
    int N, H, W;
    int Hs, Ws, Hu, Wu, Hp, Wp;     // sample grid, upsampled padded image, padded image
};

__host__ __device__ inline AugGeom aug_geom(int N, int H, int W) {
    AugGeom g;
    g.N = N; g.H = H; g.W = W;
    g.Hs = 2 * (H + 2 * AUG_HZ); g.Ws = 2 * (W + 2 * AUG_HZ);
    g.Hp = H + 2 * (H - 1); g.Wp = W + 2 * (W - 1);
    g.Hu = 2 * g.Hp; g.Wu = 2 * g.Wp;
    return g;
}

__device__ __forceinline__ bool geom_is_identity(const float* r) {
    return r[0] == 1.f && r[1] == 0.f && r[2] == 0.f && r[3] == 0.f && r[4] == 1.f && r[5] == 0.f;
}

__device__ __forceinline__ bool color_is_identity(const float* r) {
    const float* c = r + 9;
    return c[0] == 1.f && c[1] == 0.f && c[2] == 0.f && c[3] == 0.f && c[4] == 0.f && c[5] == 1.f && c[6] == 0.f &&
           c[7] == 0.f && c[8] == 0.f && c[9] == 0.f && c[10] == 1.f && c[11] == 0.f;
}

// Where sample point (i, j) reads the upsampled image U, in U's pixel index (fp64, so the large coordinates of a 256^2 U
// keep their fraction):  q = (x_s + 1/2) / 2 with x_s the centred sample coordinate, x_u = 2 G_inv q - 1/2, index
// x_u + (W_u / 2, H_u / 2) - 1/2.
struct AugMap {
    double a00, a01, a10, a11, bx, by;     // u = A (j, i) + b
};

__device__ __forceinline__ AugMap aug_map(const float* r, const AugGeom& g) {
    const double g00 = r[0], g01 = r[1], g02 = r[2], g10 = r[3], g11 = r[4], g12 = r[5];
    const double qx0 = 0.5 * (1.0 - 0.5 * g.Ws), qy0 = 0.5 * (1.0 - 0.5 * g.Hs);      // q at (i, j) = (0, 0)
    AugMap m;
    m.a00 = g00; m.a01 = g01; m.a10 = g10; m.a11 = g11;
    m.bx = 2.0 * (g00 * qx0 + g01 * qy0 + g02) + 0.5 * g.Wu - 1.0;
    m.by = 2.0 * (g10 * qx0 + g11 * qy0 + g12) + 0.5 * g.Hu - 1.0;
    return m;
}

__device__ __forceinline__ int reflect_index(int r, int n) {      // torch 'reflect' for |overhang| < n
    r = r < 0 ? -r : r;
    return r >= n ? 2 * (n - 1) - r : r;
}

// Combined weight of padded-image row t in the bilinear sample between U rows y0 (weight 1 - f) and y0 + 1 (weight f):
// U[o] = sum_t g[o + 5 - 2t] P[t] (the existing upfirdn2d's convolution with up = 2, pad = (6, 5)); rows outside U are zero.
__device__ __forceinline__ float aug_tap_weight(int t, int y0, float f, int nu) {
    float w = 0.f;
    const int m0 = y0 + 5 - 2 * t, m1 = m0 + 1;
    if (y0 >= 0 && y0 < nu && m0 >= 0 && m0 < 12) w += (1.f - f) * c_aug_g[m0];
    if (y0 + 1 >= 0 && y0 + 1 < nu && m1 >= 0 && m1 < 12) w += f * c_aug_g[m1];
    return w;
}

// S[n, i, j, c] (NHWC, 4 channels, the last zero: the FIR kernels take 4-channel pixels as one float4), one thread per
// sample point.  Images whose G_inv is exactly I get zeros when copy_identity
// is set: sae_augment_color then takes them from the input instead.
__global__ void __launch_bounds__(256)
aug_sample_kernel(const float* __restrict__ x, const float* __restrict__ rec, float* __restrict__ s, const AugGeom g,
                  int64_t xs_n, int64_t xs_c, int64_t xs_h, int64_t xs_w, int copy_identity) {
    const int64_t total = (int64_t)g.N * g.Hs * g.Ws;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(idx % g.Ws);
        const int i = (int)((idx / g.Ws) % g.Hs);
        const int n = (int)(idx / ((int64_t)g.Ws * g.Hs));
        const float* r = rec + (int64_t)n * SAE_AUG_RECORD;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        if (!(copy_identity && geom_is_identity(r))) {
            const AugMap m = aug_map(r, g);
            const double ux = m.a00 * j + m.a01 * i + m.bx, uy = m.a10 * j + m.a11 * i + m.by;
            if (ux > -1.0 && ux < (double)g.Wu && uy > -1.0 && uy < (double)g.Hu) {
                const double fx0 = floor(ux), fy0 = floor(uy);
                const int x0 = (int)fx0, y0 = (int)fy0;
                const float fx = (float)(ux - fx0), fy = (float)(uy - fy0);
                // padded rows t in [ceil((y0 - 6) / 2), floor((y0 + 6) / 2)]: at most 7
                const int ty0 = (y0 - 5) >> 1, tx0 = (x0 - 5) >> 1;
                float wy[7], wx[7];
                int ry[7], rx[7];
#pragma unroll
                for (int k = 0; k < 7; ++k) {
                    const int ty = ty0 + k, tx = tx0 + k;
                    wy[k] = (ty >= 0 && ty < g.Hp) ? aug_tap_weight(ty, y0, fy, g.Hu) : 0.f;
                    wx[k] = (tx >= 0 && tx < g.Wp) ? aug_tap_weight(tx, x0, fx, g.Wu) : 0.f;
                    ry[k] = wy[k] != 0.f ? reflect_index(ty - (g.H - 1), g.H) : 0;
                    rx[k] = wx[k] != 0.f ? reflect_index(tx - (g.W - 1), g.W) : 0;
                }
                const float* xn = x + (int64_t)n * xs_n;
#pragma unroll
                for (int ky = 0; ky < 7; ++ky) {
                    if (wy[ky] == 0.f) continue;
                    const float* row = xn + (int64_t)ry[ky] * xs_h;
                    float b0 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll
                    for (int kx = 0; kx < 7; ++kx) {
                        if (wx[kx] == 0.f) continue;
                        const float* px = row + (int64_t)rx[kx] * xs_w;
                        b0 = fmaf(wx[kx], __ldg(px), b0);
                        b1 = fmaf(wx[kx], __ldg(px + xs_c), b1);
                        b2 = fmaf(wx[kx], __ldg(px + 2 * xs_c), b2);
                    }
                    a0 = fmaf(wy[ky], b0, a0);
                    a1 = fmaf(wy[ky], b1, a1);
                    a2 = fmaf(wy[ky], b2, a2);
                }
            }
        }
        reinterpret_cast<float4*>(s)[idx] = make_float4(a0, a1, a2, 0.f);
    }
}

// Adjoint of aug_sample_kernel in gather form: dx[n, y, x, c] (NHWC) = sum over the padded-image copies (ty, tx) of input
// pixel (y, x) (reflection puts up to three per axis into P) and over the sample points (i, j) whose bilinear foot lands on
// a U pixel that ty / tx feeds:  w_y * w_x * dS[n, i, j, c].  Sample -> U coordinates are affine, so the sample points that
// can touch copy (ty, tx) lie in the preimage of a U box: bracket it generously by inverting the map, then test each point
// exactly with the forward's own arithmetic.  Images whose G_inv is exactly I copy gc (with copy_identity).
__global__ void __launch_bounds__(256)
aug_sample_adjoint_kernel(const float* __restrict__ ds, const float* __restrict__ gc, const float* __restrict__ rec,
                          float* __restrict__ dx, const AugGeom g, int copy_identity) {
    const int64_t total = (int64_t)g.N * g.H * g.W;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int xx = (int)(idx % g.W);
        const int yy = (int)((idx / g.W) % g.H);
        const int n = (int)(idx / ((int64_t)g.W * g.H));
        const float* r = rec + (int64_t)n * SAE_AUG_RECORD;
        float* o = dx + idx * 3;
        if (copy_identity && geom_is_identity(r)) {
            const float4 g4 = reinterpret_cast<const float4*>(gc)[idx];
            o[0] = g4.x; o[1] = g4.y; o[2] = g4.z;
            continue;
        }
        const AugMap m = aug_map(r, g);
        const double det = m.a00 * m.a11 - m.a01 * m.a10;
        const double i00 = m.a11 / det, i01 = -m.a01 / det, i10 = -m.a10 / det, i11 = m.a00 / det;
        int tys[3], txs[3], nty = 1, ntx = 1;
        tys[0] = yy + (g.H - 1);
        if (yy > 0) tys[nty++] = (g.H - 1) - yy;
        if (yy < g.H - 1) tys[nty++] = 3 * (g.H - 1) - yy;
        txs[0] = xx + (g.W - 1);
        if (xx > 0) txs[ntx++] = (g.W - 1) - xx;
        if (xx < g.W - 1) txs[ntx++] = 3 * (g.W - 1) - xx;
        const float4* dsn = reinterpret_cast<const float4*>(ds) + (int64_t)n * g.Hs * g.Ws;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int cy = 0; cy < nty; ++cy) {
            const int ty = tys[cy];
            for (int cx = 0; cx < ntx; ++cx) {
                const int tx = txs[cx];
                // U box of the samples whose foot can involve (ty, tx): floor(u) in [2t - 6, 2t + 6], widened by one
                const double ulo = 2.0 * tx - 7.0, uhi = 2.0 * tx + 8.0, vlo = 2.0 * ty - 7.0, vhi = 2.0 * ty + 8.0;
                double jlo = 1e300, jhi = -1e300, ilo = 1e300, ihi = -1e300;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double du = ((k & 1) ? uhi : ulo) - m.bx, dv = ((k & 2) ? vhi : vlo) - m.by;
                    const double jj = i00 * du + i01 * dv, ii = i10 * du + i11 * dv;
                    jlo = fmin(jlo, jj); jhi = fmax(jhi, jj); ilo = fmin(ilo, ii); ihi = fmax(ihi, ii);
                }
                const int j0 = (int)fmax(floor(jlo) - 1.0, 0.0), j1 = (int)fmin(ceil(jhi) + 1.0, (double)(g.Ws - 1));
                const int i0 = (int)fmax(floor(ilo) - 1.0, 0.0), i1 = (int)fmin(ceil(ihi) + 1.0, (double)(g.Hs - 1));
                for (int i = i0; i <= i1; ++i) {
                    for (int j = j0; j <= j1; ++j) {
                        const double ux = m.a00 * j + m.a01 * i + m.bx, uy = m.a10 * j + m.a11 * i + m.by;
                        if (!(ux > -1.0 && ux < (double)g.Wu && uy > -1.0 && uy < (double)g.Hu)) continue;
                        const double fx0 = floor(ux), fy0 = floor(uy);
                        const int x0 = (int)fx0, y0 = (int)fy0;
                        if (y0 < 2 * ty - 6 || y0 > 2 * ty + 6 || x0 < 2 * tx - 6 || x0 > 2 * tx + 6) continue;
                        const float wy = aug_tap_weight(ty, y0, (float)(uy - fy0), g.Hu);
                        const float wx = aug_tap_weight(tx, x0, (float)(ux - fx0), g.Wu);
                        if (wy == 0.f || wx == 0.f) continue;
                        const float w = wy * wx;
                        const float4 d = __ldg(dsn + (int64_t)i * g.Ws + j);
                        a0 = fmaf(w, d.x, a0);
                        a1 = fmaf(w, d.y, a1);
                        a2 = fmaf(w, d.z, a2);
                    }
                }
            }
        }
        o[0] = a0; o[1] = a1; o[2] = a2;
    }
}

// ------------------------------------------------------------------------------------------------- colour
// out[n, y, x, :] (NHWC) = C[:3, :3] v + offset * C[:3, 3], v = a[n, :, y, x] (strided) when copy_identity and G_inv is
// exactly I, else b[n, y, x, 0:3] (NHWC, 4 channels).  A C that is exactly I copies v.
__global__ void __launch_bounds__(256)
aug_color_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ rec,
                 float* __restrict__ out, int N, int H, int W, int64_t as_n, int64_t as_c, int64_t as_h, int64_t as_w,
                 int offset, int copy_identity) {
    const int64_t total = (int64_t)N * H * W;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int xx = (int)(idx % W);
        const int yy = (int)((idx / W) % H);
        const int n = (int)(idx / ((int64_t)W * H));
        const float* r = rec + (int64_t)n * SAE_AUG_RECORD;
        float v0, v1, v2;
        if (copy_identity && geom_is_identity(r)) {
            const float* p = a + n * as_n + yy * as_h + xx * as_w;
            v0 = __ldg(p); v1 = __ldg(p + as_c); v2 = __ldg(p + 2 * as_c);
        } else {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(b) + idx);
            v0 = b4.x; v1 = b4.y; v2 = b4.z;
        }
        float* o = out + idx * 3;
        if (color_is_identity(r)) {
            o[0] = v0; o[1] = v1; o[2] = v2;
            continue;
        }
        const float* c = r + 9;
        o[0] = fmaf(c[0], v0, fmaf(c[1], v1, fmaf(c[2], v2, offset ? c[3] : 0.f)));
        o[1] = fmaf(c[4], v0, fmaf(c[5], v1, fmaf(c[6], v2, offset ? c[7] : 0.f)));
        o[2] = fmaf(c[8], v0, fmaf(c[9], v1, fmaf(c[10], v2, offset ? c[11] : 0.f)));
    }
}

// gc[n, y, x, :] (NHWC, 4 channels, the last zero) = C[:3, :3]^T dy[n, :, y, x] (strided)
__global__ void __launch_bounds__(256)
aug_color_adjoint_kernel(const float* __restrict__ dy, const float* __restrict__ rec, float* __restrict__ gc, int N, int H,
                         int W, int64_t ds_n, int64_t ds_c, int64_t ds_h, int64_t ds_w) {
    const int64_t total = (int64_t)N * H * W;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int xx = (int)(idx % W);
        const int yy = (int)((idx / W) % H);
        const int n = (int)(idx / ((int64_t)W * H));
        const float* r = rec + (int64_t)n * SAE_AUG_RECORD;
        const float* p = dy + n * ds_n + yy * ds_h + xx * ds_w;
        const float d0 = __ldg(p), d1 = __ldg(p + ds_c), d2 = __ldg(p + 2 * ds_c);
        float4* o = reinterpret_cast<float4*>(gc) + idx;
        if (color_is_identity(r)) {
            *o = make_float4(d0, d1, d2, 0.f);
            continue;
        }
        const float* c = r + 9;
        *o = make_float4(fmaf(c[0], d0, fmaf(c[4], d1, c[8] * d2)), fmaf(c[1], d0, fmaf(c[5], d1, c[9] * d2)),
                         fmaf(c[2], d0, fmaf(c[6], d1, c[10] * d2)), 0.f);
    }
}

// ------------------------------------------------------------------------------------------------- p adjustment
__global__ void ada_adjust_kernel(float* __restrict__ p, double* __restrict__ acc, double step, double target) {
    if (acc[2] > 0.0) {
        const double rt = acc[1] / acc[2];
        const double adjust = (rt > target ? 1.0 : (rt < target ? -1.0 : 0.0)) * step;
        *p = fmaxf(0.f, *p + (float)adjust);
    }
    acc[0] = acc[1] = acc[2] = acc[3] = 0.0;
}

static inline unsigned aug_grid(int64_t work) {
    int64_t blocks = (work + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace sae

using namespace sae;

static int aug_shape(int N, int H, int W, const char* who) {
    if (N < 0 || H < 2 || W < 2) return fail(SAE_E_INVALID, "%s: bad shape N = %d, H = %d, W = %d (H, W >= 2)", who, N, H, W);
    if ((int64_t)2 * (3 * H - 2) >= ((int64_t)1 << 30) || (int64_t)2 * (3 * W - 2) >= ((int64_t)1 << 30))
        return fail(SAE_E_INVALID, "%s: image too large", who);
    return SAE_OK;
}

extern "C" int sae_augment_params(const float* u, const float* z, const float* p, float* rec, int N, int H, int W,
                                  void* stream) {
    int rc = aug_shape(N, H, W, "augment_params");
    if (rc) return rc;
    if (N == 0) return SAE_OK;
    if (!u || !z || !p || !rec) return fail(SAE_E_INVALID, "augment_params: null pointer");
    aug_params_kernel<<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(u, z, p, rec, N, H, W);
    return check_launch("augment_params");
}

extern "C" int sae_augment_sample(const float* x, const float* rec, float* s, int N, int H, int W, int64_t xs_n, int64_t xs_c,
                                  int64_t xs_h, int64_t xs_w, int copy_identity, void* stream) {
    int rc = aug_shape(N, H, W, "augment_sample");
    if (rc) return rc;
    if (N == 0) return SAE_OK;
    if (!x || !rec || !s || (reinterpret_cast<uintptr_t>(s) & 15)) return fail(SAE_E_INVALID, "augment_sample: null / unaligned pointer");
    if (xs_n < 0 || xs_c < 0 || xs_h < 0 || xs_w < 0) return fail(SAE_E_INVALID, "augment_sample: negative stride");
    const AugGeom g = aug_geom(N, H, W);
    aug_sample_kernel<<<aug_grid((int64_t)N * g.Hs * g.Ws), 256, 0, (cudaStream_t)stream>>>(x, rec, s, g, xs_n, xs_c, xs_h,
                                                                                            xs_w, copy_identity);
    return check_launch("augment_sample");
}

extern "C" int sae_augment_sample_adjoint(const float* ds, const float* gc, const float* rec, float* dx, int N, int H, int W,
                                          int copy_identity, void* stream) {
    int rc = aug_shape(N, H, W, "augment_sample_adjoint");
    if (rc) return rc;
    if (N == 0) return SAE_OK;
    if (!ds || !rec || !dx || (copy_identity && !gc) || ((reinterpret_cast<uintptr_t>(ds) | reinterpret_cast<uintptr_t>(gc)) & 15))
        return fail(SAE_E_INVALID, "augment_sample_adjoint: null / unaligned pointer");
    const AugGeom g = aug_geom(N, H, W);
    aug_sample_adjoint_kernel<<<aug_grid((int64_t)N * H * W), 256, 0, (cudaStream_t)stream>>>(ds, gc, rec, dx, g, copy_identity);
    return check_launch("augment_sample_adjoint");
}

extern "C" int sae_augment_color(const float* a, const float* b, const float* rec, float* out, int N, int H, int W,
                                 int64_t as_n, int64_t as_c, int64_t as_h, int64_t as_w, int offset, int copy_identity,
                                 void* stream) {
    if (N < 0 || H < 1 || W < 1) return fail(SAE_E_INVALID, "augment_color: bad shape");
    if (N == 0) return SAE_OK;
    if (!b || !rec || !out || (copy_identity && !a) || (reinterpret_cast<uintptr_t>(b) & 15))
        return fail(SAE_E_INVALID, "augment_color: null / unaligned pointer");
    if (as_n < 0 || as_c < 0 || as_h < 0 || as_w < 0) return fail(SAE_E_INVALID, "augment_color: negative stride");
    aug_color_kernel<<<aug_grid((int64_t)N * H * W), 256, 0, (cudaStream_t)stream>>>(a, b, rec, out, N, H, W, as_n, as_c, as_h,
                                                                                    as_w, offset, copy_identity);
    return check_launch("augment_color");
}

extern "C" int sae_augment_color_adjoint(const float* dy, const float* rec, float* gc, int N, int H, int W, int64_t ds_n,
                                         int64_t ds_c, int64_t ds_h, int64_t ds_w, void* stream) {
    if (N < 0 || H < 1 || W < 1) return fail(SAE_E_INVALID, "augment_color_adjoint: bad shape");
    if (N == 0) return SAE_OK;
    if (!dy || !rec || !gc || (reinterpret_cast<uintptr_t>(gc) & 15))
        return fail(SAE_E_INVALID, "augment_color_adjoint: null / unaligned pointer");
    if (ds_n < 0 || ds_c < 0 || ds_h < 0 || ds_w < 0) return fail(SAE_E_INVALID, "augment_color_adjoint: negative stride");
    aug_color_adjoint_kernel<<<aug_grid((int64_t)N * H * W), 256, 0, (cudaStream_t)stream>>>(dy, rec, gc, N, H, W, ds_n, ds_c,
                                                                                            ds_h, ds_w);
    return check_launch("augment_color_adjoint");
}

extern "C" int sae_ada_adjust(float* p, double* acc, double step, double target, void* stream) {
    if (!p || !acc) return fail(SAE_E_INVALID, "ada_adjust: null pointer");
    if (!std::isfinite(step) || step < 0.0 || !std::isfinite(target)) return fail(SAE_E_INVALID, "ada_adjust: bad step / target");
    ada_adjust_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(p, acc, step, target);
    return check_launch("ada_adjust");
}
