"""TEST INFRASTRUCTURE — an fp64 restatement of the adaptive discriminator augmentation (INTEGRATION.md §2h) in plain torch
ops (on the CPU, or on the GPU for speed), formulated independently of the fused kernels: the per-image matrices from the draws, the geometric chain as
``F.pad`` (reflect) -> the oracle's FIR (2x up) -> ``F.affine_grid`` + ``F.grid_sample`` -> the oracle's FIR (2x down), and
the colour matrix.  The reference has no augmentation, so there is no golden file for it; the host and GPU tests compare
the product against this."""
import math

import torch
import torch.nn.functional as F

from oracle import sae_oracle as O

SYM6 = [0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
        0.787641141030194, 0.3379294217276218, -0.07263752278646252, -0.021060292512300564, 0.04472490177066578,
        0.0017677118642428036, -0.007800708325034148]
HZ_PAD = 3
UNIFORMS, NORMALS, RECORD = 21, 7, 32


def sym6(dtype=torch.float64):
    f = torch.tensor(SYM6, dtype=torch.float64)
    return (f / f.sum()).to(dtype)


# ------------------------------------------------------------------------------------------------------------- matrices
def _eye(n, k):
    return torch.eye(k, dtype=torch.float64).expand(n, k, k).clone()


def _scale2d(sx, sy):
    m = _eye(sx.numel(), 3)
    m[:, 0, 0], m[:, 1, 1] = sx, sy
    return m


def _translate2d(tx, ty):
    m = _eye(tx.numel(), 3)
    m[:, 0, 2], m[:, 1, 2] = tx, ty
    return m


def _rotate2d(t):
    m = _eye(t.numel(), 3)
    m[:, 0, 0], m[:, 0, 1], m[:, 1, 0], m[:, 1, 1] = t.cos(), -t.sin(), t.sin(), t.cos()
    return m


def _gated(gate, m):
    """the factor where the gate is open, I elsewhere"""
    return torch.where(gate.view(-1, 1, 1), m, _eye(m.shape[0], m.shape[1]))


def matrices(u, z, p, h, w):
    """(G_inv [N, 3, 3], C [N, 4, 4]) in fp64 from the draws u [N, 21], z [N, 7] and the probability p, for h x w images.
    The column layout is the product's (csrc/augment.cu, aug_params_kernel)."""
    u, z = u.double(), z.double()
    n = u.shape[0]
    p = float(p)
    p_rot = 1.0 - math.sqrt(min(max(1.0 - p, 0.0), 1.0))
    one = torch.ones(n, dtype=torch.float64)
    G = _eye(n, 3)
    G = G @ _gated(u[:, 0] < p, _scale2d(1 - 2 * torch.floor(2 * u[:, 1]), one))
    G = G @ _gated(u[:, 2] < p, _rotate2d(math.pi / 2 * torch.floor(4 * u[:, 3])))
    G = G @ _gated(u[:, 4] < p, _translate2d(-torch.round((2 * u[:, 5] - 1) * 0.125 * w),
                                              -torch.round((2 * u[:, 6] - 1) * 0.125 * h)))
    s = torch.exp2(0.2 * z[:, 0])
    G = G @ _gated(u[:, 7] < p, _scale2d(1 / s, 1 / s))
    G = G @ _gated(u[:, 8] < p_rot, _rotate2d((2 * u[:, 9] - 1) * math.pi))
    s = torch.exp2(0.2 * z[:, 1])
    G = G @ _gated(u[:, 10] < p, _scale2d(1 / s, s))
    G = G @ _gated(u[:, 11] < p_rot, _rotate2d((2 * u[:, 12] - 1) * math.pi))
    G = G @ _gated(u[:, 13] < p, _translate2d(-0.125 * z[:, 2] * w, -0.125 * z[:, 3] * h))

    v = torch.tensor([1.0, 1.0, 1.0, 0.0], dtype=torch.float64) / math.sqrt(3.0)
    vv = torch.outer(v, v)
    I4 = _eye(n, 4)
    C = _eye(n, 4)
    b = 0.2 * z[:, 4]
    f = _eye(n, 4)
    f[:, 0, 3] = f[:, 1, 3] = f[:, 2, 3] = b
    C = _gated(u[:, 14] < p, f) @ C
    c = torch.exp2(0.5 * z[:, 5])
    f = _eye(n, 4)
    f[:, 0, 0] = f[:, 1, 1] = f[:, 2, 2] = c
    C = _gated(u[:, 15] < p, f) @ C
    i = torch.floor(2 * u[:, 16 + 1])
    C = _gated(u[:, 16] < p, I4 - 2 * vv * i.view(-1, 1, 1)) @ C
    t = (2 * u[:, 19] - 1) * math.pi
    # Rodrigues: I cos t + sin t [v]x + (1 - cos t) v v^T on the rgb block
    k = torch.zeros(4, 4, dtype=torch.float64)
    a = v[0].item()
    k[0, 1], k[0, 2], k[1, 0], k[1, 2], k[2, 0], k[2, 1] = -a, a, a, -a, -a, a
    rot = torch.zeros(n, 4, 4, dtype=torch.float64)
    eye3 = torch.diag(torch.tensor([1.0, 1.0, 1.0, 0.0], dtype=torch.float64))
    rot += eye3 * t.cos().view(-1, 1, 1) + k * t.sin().view(-1, 1, 1) + vv * (1 - t.cos()).view(-1, 1, 1)
    rot[:, 3, 3] = 1.0
    C = _gated(u[:, 18] < p, rot) @ C
    s = torch.exp2(z[:, 6])
    C = _gated(u[:, 20] < p, vv + (I4 - vv) * s.view(-1, 1, 1)) @ C
    return G, C


def pack(G, C):
    """the product's per-image record [N, 32]: G_inv row-major, C row-major, zeros (fp32 unless G is fp64 already)"""
    n = G.shape[0]
    rec = torch.zeros(n, RECORD, dtype=G.dtype)
    rec[:, :9] = G.reshape(n, 9)
    rec[:, 9:25] = C.reshape(n, 16).to(G.dtype)
    return rec


def unpack(rec):
    n = rec.shape[0]
    return rec[:, :9].reshape(n, 3, 3), rec[:, 9:25].reshape(n, 4, 4)


def is_identity(G):
    """[N] bool: G_inv exactly I (the rows the transform uses)"""
    eye = torch.eye(3, dtype=G.dtype, device=G.device)[:2]
    return (G[:, :2] == eye).all(dim=2).all(dim=1)


# ------------------------------------------------------------------------------------------------------------- operator
def sample(x, G):
    """steps 1-3: [N, C, H, W] -> the sample grid [N, C, 2(H + 6), 2(W + 6)] (every image resampled)"""
    n, c, h, w = x.shape
    f = sym6(x.dtype).to(x.device)
    P = F.pad(x, (w - 1, w - 1, h - 1, h - 1), mode="reflect")
    U = O.upfirdn2d(P, torch.outer(f, f) * 4, up=2, pad=(6, 5))
    hu, wu = U.shape[2], U.shape[3]
    hs, ws = 2 * (h + 2 * HZ_PAD), 2 * (w + 2 * HZ_PAD)
    # normalised sample coordinate (align_corners=False) -> normalised U coordinate: x_s = xn * W_s / 2, U index = x_u +
    # W_u / 2 - 1/2 with x_u = A (x_s + 1/2) + 2 t - 1/2, i.e. un = 2 x_u / W_u
    G = G.to(x)
    A, t = G[:, :2, :2], G[:, :2, 2]
    theta = torch.zeros(n, 2, 3, dtype=x.dtype, device=x.device)
    size = torch.tensor([wu, hu], dtype=x.dtype, device=x.device).view(1, 2)
    theta[:, :, 0] = A[:, :, 0] * (ws / 2)
    theta[:, :, 1] = A[:, :, 1] * (hs / 2)
    theta[:, :, 2] = 0.5 * A.sum(2) + 2 * t - 0.5
    theta = theta * (2 / size).view(1, 2, 1)
    grid = F.affine_grid(theta, (n, c, hs, ws), align_corners=False)
    return F.grid_sample(U, grid, mode="bilinear", padding_mode="zeros", align_corners=False)


def downsample(s):
    """step 4: upfirdn2d(S, flip(f) (x) flip(f), down=2, pad=(-1, -1))"""
    f = torch.flip(sym6(s.dtype), [0]).to(s.device)
    return O.upfirdn2d(s, torch.outer(f, f), down=2, pad=(-1, -1))


def geometric(x, G, copy_identity=True):
    out = downsample(sample(x, G))
    if copy_identity:
        out = torch.where(is_identity(G).view(-1, 1, 1, 1), x, out)
    return out


class _Geometric(torch.autograd.Function):
    """``geometric`` with a backward that is differentiable again: the operator is linear, so its backward is its adjoint
    (first-order autograd of ``geometric``) and the adjoint's backward is the operator.  torch's grid_sample has no double
    backward, and R1 differentiates twice."""

    @staticmethod
    def forward(ctx, x, G, copy_identity):
        ctx.save_for_backward(G)
        ctx.copy_identity = copy_identity
        return geometric(x, G, copy_identity)

    @staticmethod
    def backward(ctx, g):
        G, = ctx.saved_tensors
        return _GeometricAdjoint.apply(g, G, ctx.copy_identity), None, None


class _GeometricAdjoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, g, G, copy_identity):
        ctx.save_for_backward(G)
        ctx.copy_identity = copy_identity
        x0 = torch.zeros_like(g).requires_grad_()
        with torch.enable_grad():
            y = geometric(x0, G, copy_identity)
        return torch.autograd.grad(y, x0, g)[0]

    @staticmethod
    def backward(ctx, gg):
        G, = ctx.saved_tensors
        return _Geometric.apply(gg, G, ctx.copy_identity), None, None


def color(x, C, offset=True):
    C = C.to(x)
    y = torch.einsum("nij,njhw->nihw", C[:, :3, :3], x)
    if offset:
        y = y + C[:, :3, 3].view(-1, 3, 1, 1)
    return y


def augment(x, G, C, copy_identity=True):
    """the whole operator; twice differentiable in x"""
    return color(_Geometric.apply(x, G, copy_identity), C)
