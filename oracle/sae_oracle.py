"""ORACLE — test infrastructure only.  CPU restatement of the Swapping-Autoencoder training hot path.

This file is the checker for the CUDA product in ``swapping_autoencoder_pytorch_b200/``; nothing in the product
imports it.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl reference``
legs may import it.  It restates, in a functional style over a flat ``{state_dict key: tensor}`` parameter
dictionary, the algorithm of the reference (taesungp/swapping-autoencoder-pytorch @ 6baa180) for the path named
in BASELINE.json; every function cites the reference lines it follows (paths relative to the reference root).

Arithmetic: plain PyTorch CPU ops in whatever dtype the inputs carry (fp32 for timing, fp64 for tight parity and
gradcheck), exactly the arithmetic library the reference's own native fallback uses (``upfirdn2d_native``,
upfirdn2d.py:162-222; ``F.leaky_relu(input + bias) * scale``, fused_act.py:93-96).  ``fir_numpy`` is an
independent direct-summation NumPy restatement of the FIR used to pin the torch formulation.

PARITY PINNING: the reference ships no tests or golden vectors (SURVEY.md §4).  The oracle is pinned against the
reference itself, imported in the build container by ``oracle/make_golden.py`` (native-PyTorch path, fp64), which
commits small input/output fixtures under ``tests/golden/``; ``tests/test_oracle_golden.py`` replays them.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

SQRT2 = math.sqrt(2.0)


# =====================================================================================================
# custom ops
# =====================================================================================================
def fir_numpy(x, k, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0)):
    """Direct-summation upfirdn2d on a NumPy array [B,C,H,W]; pad = (x0, x1, y0, y1).
    out[oy,ox] = sum_{ky,kx} k[kh-1-ky, kw-1-kx] * U[oy*down_y + ky, ox*down_x + kx], with U the zero-inserted,
    padded (negative pad crops) input — the same definition the reference CUDA kernel implements
    (upfirdn2d_kernel.cu:52-137) and its native fallback emulates (upfirdn2d.py:162-222)."""
    x = np.asarray(x)
    k = np.asarray(k)
    b, c, h, w = x.shape
    kh, kw = k.shape
    ux, uy = up
    dx, dy = down
    px0, px1, py0, py1 = pad
    U = np.zeros((b, c, h * uy, w * ux), dtype=x.dtype)
    U[:, :, ::uy, ::ux] = x
    U = np.pad(U, ((0, 0), (0, 0), (max(py0, 0), max(py1, 0)), (max(px0, 0), max(px1, 0))))
    U = U[:, :, max(-py0, 0):U.shape[2] - max(-py1, 0), max(-px0, 0):U.shape[3] - max(-px1, 0)]
    fh, fw = U.shape[2] - kh + 1, U.shape[3] - kw + 1
    full = np.zeros((b, c, fh, fw), dtype=x.dtype)
    for ky in range(kh):
        for kx in range(kw):
            full += k[kh - 1 - ky, kw - 1 - kx] * U[:, :, ky:ky + fh, kx:kx + fw]
    return full[:, :, ::dy, ::dx]


def upfirdn2d(x, k, up=1, down=1, pad=(0, 0)):
    """Differentiable torch formulation, same pad on x and y (reference upfirdn2d.py:150-222)."""
    b, c, h, w = x.shape
    kh, kw = k.shape
    p0, p1 = pad
    u = x.reshape(b * c, 1, h, 1, w, 1)
    if up > 1:
        u = F.pad(u, [0, up - 1, 0, 0, 0, up - 1])
    u = u.reshape(b * c, 1, h * up, w * up)
    u = F.pad(u, [max(p0, 0), max(p1, 0), max(p0, 0), max(p1, 0)])
    u = u[:, :, max(-p0, 0):u.shape[2] - max(-p1, 0), max(-p0, 0):u.shape[3] - max(-p1, 0)]
    out = F.conv2d(u, torch.flip(k, [0, 1]).to(x).view(1, 1, kh, kw))
    out = out[:, :, ::down, ::down]
    return out.reshape(b, c, out.shape[2], out.shape[3])


def fused_leaky_relu(x, bias, negative_slope=0.2, scale=SQRT2):
    """lrelu(x + b[c]) * scale, bias on dim 1 (reference fused_act.py:89-96; kernel switch
    fused_bias_act_kernel.cu:36-45)."""
    if bias is not None:
        x = x + bias.view(1, -1, *([1] * (x.dim() - 2)))
    return F.leaky_relu(x, negative_slope) * scale


def make_kernel(taps, dtype=torch.float32):
    """reference stylegan2_layers.py:27-35"""
    k = torch.tensor(taps, dtype=dtype)
    if k.dim() == 1:
        k = k[None, :] * k[:, None]
    return k / k.sum()


def normalize(v):
    """reference util/util.py:18-22"""
    return v * torch.rsqrt(torch.sum(v ** 2, dim=1, keepdim=True) + 1e-8)


# =====================================================================================================
# layers (functional; P maps state_dict keys to tensors)
# =====================================================================================================
def equal_conv2d(P, name, x, stride=1, padding=0):
    """reference stylegan2_layers.py:115-142"""
    w = P[name + ".weight"]
    scale = 1.0 / math.sqrt(w.shape[1] * w.shape[2] * w.shape[3])
    return F.conv2d(x, w * scale, bias=P.get(name + ".bias"), stride=stride, padding=padding)


def equal_linear(P, name, x, activation=False, lr_mul=1.0):
    """reference stylegan2_layers.py:153-188 (2-D inputs and the 4-D 1x1-conv branch)"""
    w = P[name + ".weight"]
    scale = (1.0 / math.sqrt(w.shape[1])) * lr_mul
    bias = P.get(name + ".bias")
    b = bias * lr_mul if bias is not None else None
    if x.dim() > 2:
        out = F.conv2d(x, (w * scale)[:, :, None, None])
    else:
        out = F.linear(x, w * scale)
    if activation:
        return fused_leaky_relu(out, b)
    if b is not None:
        out = out + (b.view(1, -1, 1, 1) if out.dim() > 2 else b)
    return out


def conv_layer(P, name, x, kernel_size, downsample=False, blur_taps=(1, 3, 3, 1), bias=True, activate=True, pad=None,
               reflection_pad=False):
    """[Blur | RefPad] -> Conv -> [Act]  (reference stylegan2_layers.py:612-668; FIR pads :628-634)."""
    if downsample:
        p = (len(blur_taps) - 2) + (kernel_size - 1) if pad is None else pad
        p0, p1 = (p + 1) // 2, p // 2
        k = P.get(name + ".Blur.kernel")
        if k is None:
            k = make_kernel(list(blur_taps), x.dtype)
        if reflection_pad:
            x = F.pad(x, (p0, p1, p0, p1), mode="reflect")
            p0 = p1 = 0
        x = upfirdn2d(x, k.to(x), pad=(p0, p1))
        stride, padding = 2, 0
    else:
        stride = 1
        padding = kernel_size // 2 if pad is None else pad
        if reflection_pad:
            x = F.pad(x, (padding,) * 4, mode="reflect")
            padding = 0
    x = equal_conv2d(P, name + ".Conv", x, stride=stride, padding=padding)
    if activate:
        if bias:
            x = fused_leaky_relu(x, P[name + ".Act.bias"])
        else:
            x = F.leaky_relu(x, 0.2) * SQRT2
    return x


def res_block(P, name, x, blur_taps=(1, 3, 3, 1), reflection_pad=False, pad=None, downsample=True):
    """reference stylegan2_layers.py:672-693"""
    out = conv_layer(P, name + ".conv1", x, 3, reflection_pad=reflection_pad, pad=pad)
    out = conv_layer(P, name + ".conv2", out, 3, downsample=downsample, blur_taps=blur_taps,
                     reflection_pad=reflection_pad, pad=pad)
    skip = conv_layer(P, name + ".skip", x, 1, downsample=downsample, blur_taps=blur_taps, activate=False, bias=False)
    return (out + skip) / SQRT2


def modulated_conv2d(P, name, x, style, kernel_size, demodulate=True, upsample=False, blur_taps=(1, 3, 3, 1)):
    """reference stylegan2_layers.py:266-325 with new_demodulation (:258): RMS-normalised style scales the input,
    one per-output-channel-normalised filter for the whole batch (the reference's weight.repeat + groups=batch
    grouped conv computes exactly this — SURVEY.md §0.1)."""
    w = P[name + ".weight"][0]                              # [Cout, Cin, k, k]
    cin = w.shape[1]
    s = equal_linear(P, name + ".modulation", style.reshape(style.shape[0], -1))
    if demodulate:
        s = s * torch.rsqrt(s.pow(2).mean(dim=1, keepdim=True) + 1e-8)
    x = x * s.view(-1, cin, 1, 1)
    w = w * (1.0 / math.sqrt(cin * kernel_size ** 2))
    if demodulate:
        w = w * torch.rsqrt(w.pow(2).sum(dim=(1, 2, 3), keepdim=True) + 1e-8)
    if upsample:
        out = F.conv_transpose2d(x, w.transpose(0, 1), stride=2, padding=0)
        p = (len(blur_taps) - 2) - (kernel_size - 1)
        k = P.get(name + ".blur.kernel")
        if k is None:
            k = make_kernel(list(blur_taps), x.dtype) * 4
        return upfirdn2d(out, k.to(x), pad=((p + 1) // 2 + 1, p // 2 + 1))
    return F.conv2d(x, w, padding=kernel_size // 2)


def styled_conv(P, name, x, style, upsample=False, use_noise=True, noise=None, blur_taps=(1, 3, 3, 1)):
    """ModulatedConv2d -> NoiseInjection -> FusedLeakyReLU  (reference stylegan2_layers.py:367-405, :328-351)"""
    out = modulated_conv2d(P, name + ".conv", x, style, 3, upsample=upsample, blur_taps=blur_taps)
    if use_noise:
        if noise is None:
            noise = torch.randn(out.shape[0], 1, out.shape[2], out.shape[3], dtype=out.dtype).to(out.device)
        out = out + P[name + ".noise.weight"] * noise
    return fused_leaky_relu(out, P[name + ".activate.bias"])


# =====================================================================================================
# networks
# =====================================================================================================
def _sub(P, prefix):
    n = len(prefix)
    return {k[n:]: v for k, v in P.items() if k.startswith(prefix)}


def encoder_nc(opt, idx):
    """reference encoder.py:87-91"""
    nc = opt.netE_nc_steepness ** (5 + idx) * opt.netE_scale_capacity
    return round(min(opt.global_code_ch, int(round(nc))))


def encoder_forward(P, opt, x):
    """E (reference encoder.py:40-114): returns (sp, gl), both L2-normalised over dim 1."""
    blur = (1, 2, 1) if opt.use_antialias else (1,)
    h = conv_layer(P, "FromRGB", x, 1)
    for i in range(opt.netE_num_downsampling_sp):
        h = res_block(P, "DownToSpatialCode.ResBlockDownBy%d" % (2 ** i), h, blur_taps=blur, reflection_pad=True)
    sp = conv_layer(P, "ToSpatialCode.0", h, 1, activate=True, bias=True)
    sp = conv_layer(P, "ToSpatialCode.1", sp, 1, activate=False, bias=True)
    g = h
    for i in range(opt.netE_num_downsampling_gl):
        j = opt.netE_num_downsampling_sp + i
        g = conv_layer(P, "DownToGlobalCode.ConvLayerDownBy%d" % (2 ** j), g, 3, blur_taps=(1,), downsample=True, pad=0)
    gl = equal_linear(P, "ToGlobalCode.0", g.mean(dim=(2, 3)))
    return normalize(sp), normalize(gl)


def generator_nf(opt, num_up):
    """reference generator.py:141-144"""
    ch = 128 * (2 ** (opt.netE_num_downsampling_sp - num_up))
    return int(min(512, ch) * opt.netG_scale_capacity)


def generator_forward(P, opt, sp, gl, noises=None):
    """G (reference generator.py:105-161).  ``noises`` optionally maps "<block>.<conv>" to a [B,1,H,W] tensor."""
    noises = noises or {}
    blur = (1, 3, 3, 1) if opt.use_antialias else (1,)
    sp, gl = normalize(sp), normalize(gl)
    x = sp * equal_linear(P, "SpatialCodeModulation.scale", gl)[:, :, None, None] \
        + equal_linear(P, "SpatialCodeModulation.bias", gl)[:, :, None, None]
    ch = opt.spatial_code_ch
    for i in range(opt.netG_num_base_resnet_layers):
        nxt = max(opt.spatial_code_ch, round((i + 1) / opt.netG_num_base_resnet_layers * generator_nf(opt, 0)))
        name = "HeadResnetBlock%d" % i
        skip = conv_layer(P, name + ".skip", x, 1, activate=False, bias=False) if ch != nxt else x
        r = styled_conv(P, name + ".conv1", x, gl, noise=noises.get(name + ".conv1"))
        r = styled_conv(P, name + ".conv2", r, gl, noise=noises.get(name + ".conv2"))
        x = (skip + r) / SQRT2
        ch = nxt
    for j in range(opt.netE_num_downsampling_sp):
        nxt = generator_nf(opt, j + 1)
        name = "UpsamplingResBlock%d" % (2 ** (4 + j))
        skip = conv_layer(P, name + ".skip", x, 1, activate=True, bias=True) if ch != nxt else x
        skip = F.interpolate(skip, scale_factor=2, mode="bilinear", align_corners=False)
        r = styled_conv(P, name + ".conv1", x, gl, upsample=True, use_noise=opt.netG_use_noise,
                        noise=noises.get(name + ".conv1"), blur_taps=blur)
        r = styled_conv(P, name + ".conv2", r, gl, use_noise=opt.netG_use_noise, noise=noises.get(name + ".conv2"))
        x = (skip + r) / SQRT2
        ch = nxt
    rgb = modulated_conv2d(P, "ToRGB.conv", x, gl, 1, demodulate=False)
    return rgb + P["ToRGB.bias"]


def _d_channels(cm):
    return {4: 512, 8: 512, 16: min(512, int(512 * cm)), 32: min(512, int(512 * cm)), 64: int(256 * cm),
            128: int(128 * cm), 256: int(64 * cm), 512: int(32 * cm), 1024: int(16 * cm)}


def discriminator_features(P, opt, x):
    """D trunk (reference stylegan2_layers.py:696-745 via discriminator.py:12-17); keys relative to "stylegan2_D."."""
    blur = (1, 3, 3, 1) if opt.use_antialias else (1,)
    size = 2 ** int(round(math.log(opt.crop_size, 2)))
    log_size = int(math.log(size, 2))
    h = conv_layer(P, "stylegan2_D.convs.0", x, 1)
    for i in range(log_size, 2, -1):
        name = str(9 - i) if i <= 8 else "%dx%d" % (2 ** i, 2 ** i)
        h = res_block(P, "stylegan2_D.convs." + name, h, blur_taps=blur)
    return conv_layer(P, "stylegan2_D.final_conv", h, 3)


def discriminator_forward(P, opt, x):
    h = discriminator_features(P, opt, x)
    h = equal_linear(P, "stylegan2_D.final_linear.0", h.reshape(h.shape[0], -1), activation=True)
    return equal_linear(P, "stylegan2_D.final_linear.1", h)


def patch_extract_features(P, opt, patches, aggregate=False):
    """Dpatch trunk (reference patch_discriminator.py:103-158). patches [B,T,3,S,S] -> [B*T, C, 2, 2]"""
    b, t = patches.shape[:2]
    blur = (1, 3, 3, 1) if opt.use_antialias else (1,)
    log_size = int(math.ceil(math.log(opt.patch_size, 2)))
    h = conv_layer(P, "convs.0", patches.flatten(0, 1), 3)
    for i in range(log_size, 2, -1):
        name = str(7 - i) if i <= 6 else "%dx%d" % (2 ** i, 2 ** i)
        h = res_block(P, "convs." + name, h, blur_taps=blur)
    h = res_block(P, "convs.5", h, downsample=False)
    h = conv_layer(P, "convs.6", h, 3, pad=0)
    h = h.view(b, t, *h.shape[1:])
    if aggregate:
        h = h.mean(1, keepdim=True).expand(-1, t, -1, -1, -1)
    return h.flatten(0, 1)


def patch_discriminate(P, f1, f2):
    """reference patch_discriminator.py:167-171"""
    h = torch.cat([f1.flatten(1), f2.flatten(1)], dim=1)
    for i in range(3):
        h = equal_linear(P, "pairlinear.%d" % i, h, activation=True)
    return equal_linear(P, "pairlinear.3", h)


# =====================================================================================================
# loss graph (reference models/swapping_autoencoder_model.py) and training step
# =====================================================================================================
def gan_loss(pred, real):
    """reference models/networks/loss.py:11-16"""
    return F.softplus(-pred if real else pred).view(pred.size(0), -1).mean(dim=1)


def swap(x):
    """reference swapping_autoencoder_model.py:53-60"""
    return x.reshape(x.shape[0] // 2, 2, *x.shape[1:]).flip(1).reshape(x.shape)


def draw_crop_parameters(B, opt):
    """flip, scale, offset in the reference's draw order (util/util.py:326-336)"""
    flip = torch.round(torch.rand(B, 1, 1, 1)) * 2 - 1.0
    scale = torch.rand(B, 1, 1, 2) * (opt.patch_max_scale - opt.patch_min_scale) + opt.patch_min_scale
    offset = (torch.rand(B, 1, 1, 2) * 2 - 1) * (1 - scale)
    return flip, scale, offset


def random_crops(x, opt):
    """reference util/util.py:323-343"""
    n = opt.patch_num_crops
    size = opt.patch_size
    B = x.size(0) * n
    flip, scale, offset = (t.to(x) for t in draw_crop_parameters(B, opt))      # drawn on the host: one RNG stream
    lin = torch.linspace(-1.0, 1.0, size, dtype=x.dtype).to(x.device)
    gx = lin.view(1, 1, size, 1).expand(B, size, size, 1)
    gy = lin.view(1, size, 1, 1).expand(B, size, size, 1)
    unit = torch.cat([gx * flip, gy], dim=3)
    xx = x.unsqueeze(1).expand(-1, n, -1, -1, -1).flatten(0, 1)
    crop = F.grid_sample(xx, unit * scale + offset, align_corners=False)
    return crop.view(B // n, n, crop.size(1), crop.size(2), crop.size(3))


class OracleModel:
    """E, G, D, Dpatch parameters (reference state_dict keys) + the three loss commands."""

    def __init__(self, opt, state_dict):
        self.opt = opt
        self.E = _sub(state_dict, "E.")
        self.G = _sub(state_dict, "G.")
        self.D = _sub(state_dict, "D.")
        self.Dp = _sub(state_dict, "Dpatch.")

    def params(self, mode):
        def leaves(d):
            return [v for k, v in d.items() if not k.endswith(".kernel")]
        return leaves(self.G) + leaves(self.E) if mode == "generator" else leaves(self.D) + leaves(self.Dp)

    def autoencode(self, real):
        sp, gl = encoder_forward(self.E, self.opt, real)
        return generator_forward(self.G, self.opt, sp, gl)

    def discriminator_losses(self, real, noises=(None, None)):
        """reference swapping_autoencoder_model.py:62-136.  ``noises``: the ``generator_forward`` noise dicts of the two G
        calls (rec, mix); None draws fresh noise."""
        opt = self.opt
        b = real.size(0)
        sp, gl = encoder_forward(self.E, opt, real)
        rec = generator_forward(self.G, opt, sp[:b // 2], gl[:b // 2], noises[0])
        mix = generator_forward(self.G, opt, swap(sp), gl, noises[1])
        L = {}
        if opt.lambda_GAN > 0:
            L["D_real"] = gan_loss(discriminator_forward(self.D, opt, real), True) * opt.lambda_GAN
            L["D_rec"] = gan_loss(discriminator_forward(self.D, opt, rec), False) * (0.5 * opt.lambda_GAN)
            L["D_mix"] = gan_loss(discriminator_forward(self.D, opt, mix), False) * (0.5 * opt.lambda_GAN)
        if opt.lambda_PatchGAN > 0:
            rf = patch_extract_features(self.Dp, opt, random_crops(real, opt), aggregate=opt.patch_use_aggregation)
            tf = patch_extract_features(self.Dp, opt, random_crops(real, opt))
            mf = patch_extract_features(self.Dp, opt, random_crops(mix, opt))
            L["PatchD_real"] = gan_loss(patch_discriminate(self.Dp, rf, tf), True) * opt.lambda_PatchGAN
            L["PatchD_mix"] = gan_loss(patch_discriminate(self.Dp, rf, mf), False) * opt.lambda_PatchGAN
        return L

    def r1_loss(self, real):
        """reference swapping_autoencoder_model.py:138-185"""
        opt = self.opt
        pen = 0.0
        if opt.lambda_R1 > 0:
            real = real.detach().requires_grad_()
            pred = discriminator_forward(self.D, opt, real).sum()
            g, = torch.autograd.grad(pred, [real], create_graph=True, retain_graph=True)
            pen = g.pow(2).sum(dim=(1, 2, 3)) * (opt.lambda_R1 * 0.5)
        cpen = 0.0
        if opt.lambda_patch_R1 > 0:
            rc = random_crops(real, opt).detach().requires_grad_()
            tc = random_crops(real, opt).detach().requires_grad_()
            rf = patch_extract_features(self.Dp, opt, rc, aggregate=opt.patch_use_aggregation)
            tf = patch_extract_features(self.Dp, opt, tc)
            pred = patch_discriminate(self.Dp, rf, tf).sum()
            g1, g2 = torch.autograd.grad(pred, [rc, tc], create_graph=True, retain_graph=True)
            dims = list(range(1, g1.ndim))
            cpen = (g1.pow(2).sum(dims) + g2.pow(2).sum(dims)) * (0.5 * opt.lambda_patch_R1 * 0.5)
        return {"D_R1": pen + cpen}

    def generator_losses(self, real, noises=(None, None)):
        """reference swapping_autoencoder_model.py:187-231.  ``noises`` as in ``discriminator_losses``."""
        opt = self.opt
        b = real.size(0)
        sp, gl = encoder_forward(self.E, opt, real)
        rec = generator_forward(self.G, opt, sp[:b // 2], gl[:b // 2], noises[0])
        sp_mix = swap(sp)
        L = {}
        l1 = (rec - real[:b // 2]).abs().mean()
        if opt.lambda_L1 > 0:
            L["G_L1"] = l1 * opt.lambda_L1
        if opt.crop_size >= 1024:
            real, gl, sp_mix = real[b // 2:], gl[b // 2:], sp_mix[b // 2:]
        mix = generator_forward(self.G, opt, sp_mix, gl, noises[1])
        if opt.lambda_GAN > 0:
            L["G_GAN_rec"] = gan_loss(discriminator_forward(self.D, opt, rec), True) * (opt.lambda_GAN * 0.5)
            L["G_GAN_mix"] = gan_loss(discriminator_forward(self.D, opt, mix), True) * (opt.lambda_GAN * 1.0)
        if opt.lambda_PatchGAN > 0:
            rf = patch_extract_features(self.Dp, opt, random_crops(real, opt), aggregate=opt.patch_use_aggregation).detach()
            mf = patch_extract_features(self.Dp, opt, random_crops(mix, opt))
            L["G_mix"] = gan_loss(patch_discriminate(self.Dp, rf, mf), True) * opt.lambda_PatchGAN
        return L


class OracleTrainer:
    """D/G alternation with lazy R1 and the reference's two Adams
    (reference optimizers/swapping_autoencoder_optimizer.py:24-111)."""

    def __init__(self, model):
        self.m = model
        opt = model.opt
        self.gp = model.params("generator")
        self.dp = model.params("discriminator")
        for p in self.gp + self.dp:
            p.requires_grad_(True)
        self.opt_g = torch.optim.Adam(self.gp, lr=opt.lr, betas=(opt.beta1, opt.beta2))
        c = opt.R1_once_every / (1 + opt.R1_once_every)
        self.opt_d = torch.optim.Adam(self.dp, lr=opt.lr * c, betas=(opt.beta1 ** c, opt.beta2 ** c))
        self.calls = 0
        self.d_iters = 0

    def _req(self, g, d):
        for p in self.gp:
            p.requires_grad_(g)
        for p in self.dp:
            p.requires_grad_(d)

    def train_one_step(self, real):
        self.calls += 1
        opt = self.m.opt
        if self.calls % 2 == 1:                     # discriminator half-step first
            self._req(False, True)
            self.d_iters += 1
            self.opt_d.zero_grad()
            L = self.m.discriminator_losses(real)
            sum(v.mean() for v in L.values()).backward()
            self.opt_d.step()
            if (opt.lambda_R1 > 0 or opt.lambda_patch_R1 > 0) and self.d_iters % opt.R1_once_every == 0:
                self.opt_d.zero_grad()
                R = self.m.r1_loss(real)
                (sum(v.mean() for v in R.values()) * opt.R1_once_every).backward()
                self.opt_d.step()
                L.update(R)
        else:
            self._req(True, False)
            self.opt_g.zero_grad()
            L = self.m.generator_losses(real)
            sum(v.mean() for v in L.values()).backward()
            self.opt_g.step()
        return {k: float(v.detach().mean()) for k, v in L.items()}


def init_state_dict(opt, seed=0, dtype=torch.float32):
    """Random-init parameters with the reference's shapes, keys and init distributions (all conv / linear weights
    N(0,1), biases 0, modulation bias 1, noise weight 0 — SURVEY.md §8(d)); built from the shape table of the
    product's own modules is deliberately avoided: shapes are derived here from the option set."""
    rs = np.random.RandomState(seed)      # NumPy's legacy generator: bit-stable across versions and machines
    sd = {}

    def randn(*shape):
        return torch.from_numpy(rs.standard_normal(shape)).to(dtype)

    def conv(name, cin, cout, k, bias):
        sd[name + ".weight"] = randn(cout, cin, k, k)
        if bias:
            sd[name + ".bias"] = torch.zeros(cout, dtype=dtype)

    def lin(name, cin, cout, bias_init=0.0):
        sd[name + ".weight"] = randn(cout, cin)
        sd[name + ".bias"] = torch.full((cout,), bias_init, dtype=dtype)

    def convlayer(name, cin, cout, k, bias=True, activate=True):
        conv(name + ".Conv", cin, cout, k, bias and not activate)
        if activate and bias:
            sd[name + ".Act.bias"] = torch.zeros(cout, dtype=dtype)

    def resblock(name, cin, cout):
        convlayer(name + ".conv1", cin, cin, 3)
        convlayer(name + ".conv2", cin, cout, 3)
        convlayer(name + ".skip", cin, cout, 1, bias=False, activate=False)

    def styled(name, cin, cout, sdim):
        sd[name + ".conv.weight"] = randn(1, cout, cin, 3, 3)
        lin(name + ".conv.modulation", sdim, cin, 1.0)
        sd[name + ".noise.weight"] = torch.zeros(1, dtype=dtype)
        sd[name + ".activate.bias"] = torch.zeros(cout, dtype=dtype)

    # E
    n_sp, n_gl = opt.netE_num_downsampling_sp, opt.netE_num_downsampling_gl
    convlayer("E.FromRGB", 3, encoder_nc(opt, 0), 1)
    for i in range(n_sp):
        resblock("E.DownToSpatialCode.ResBlockDownBy%d" % (2 ** i), encoder_nc(opt, i), encoder_nc(opt, i + 1))
    ch = encoder_nc(opt, n_sp)
    convlayer("E.ToSpatialCode.0", ch, ch, 1)
    convlayer("E.ToSpatialCode.1", ch, opt.spatial_code_ch, 1, activate=False)
    for i in range(n_gl):
        j = n_sp + i
        convlayer("E.DownToGlobalCode.ConvLayerDownBy%d" % (2 ** j), encoder_nc(opt, j), encoder_nc(opt, j + 1), 3)
    lin("E.ToGlobalCode.0", encoder_nc(opt, n_sp + n_gl), opt.global_code_ch)
    # G
    sdim = opt.global_code_ch + opt.num_classes
    lin("G.SpatialCodeModulation.scale", sdim, opt.spatial_code_ch)
    lin("G.SpatialCodeModulation.bias", sdim, opt.spatial_code_ch)
    ch = opt.spatial_code_ch
    for i in range(opt.netG_num_base_resnet_layers):
        nxt = max(opt.spatial_code_ch, round((i + 1) / opt.netG_num_base_resnet_layers * generator_nf(opt, 0)))
        name = "G.HeadResnetBlock%d" % i
        styled(name + ".conv1", ch, nxt, sdim)
        styled(name + ".conv2", nxt, nxt, sdim)
        if ch != nxt:
            convlayer(name + ".skip", ch, nxt, 1, bias=False, activate=False)
        ch = nxt
    for j in range(n_sp):
        nxt = generator_nf(opt, j + 1)
        name = "G.UpsamplingResBlock%d" % (2 ** (4 + j))
        styled(name + ".conv1", ch, nxt, sdim)
        styled(name + ".conv2", nxt, nxt, sdim)
        if ch != nxt:
            convlayer(name + ".skip", ch, nxt, 1)
        ch = nxt
    sd["G.ToRGB.conv.weight"] = randn(1, 3, ch, 1, 1)
    lin("G.ToRGB.conv.modulation", sdim, ch, 1.0)
    sd["G.ToRGB.bias"] = torch.zeros(1, 3, 1, 1, dtype=dtype)
    # D
    chans = _d_channels(2.0 * opt.netD_scale_capacity)
    size = 2 ** int(round(math.log(opt.crop_size, 2)))
    log_size = int(math.log(size, 2))
    convlayer("D.stylegan2_D.convs.0", 3, chans[size], 1)
    ch = chans[size]
    for i in range(log_size, 2, -1):
        nxt = chans[2 ** (i - 1)]
        name = str(9 - i) if i <= 8 else "%dx%d" % (2 ** i, 2 ** i)
        resblock("D.stylegan2_D.convs." + name, ch, nxt)
        ch = nxt
    convlayer("D.stylegan2_D.final_conv", ch, chans[4], 3)
    side = int(4 * opt.crop_size / size)
    lin("D.stylegan2_D.final_linear.0", chans[4] * side * side, chans[4])
    lin("D.stylegan2_D.final_linear.1", chans[4], 1)
    # Dpatch
    cm, cap = opt.netPatchD_scale_capacity, opt.netPatchD_max_nc
    pch = {4: min(cap, int(256 * cm)), 8: min(cap, int(128 * cm)), 16: min(cap, int(64 * cm)), 32: int(32 * cm),
           64: int(16 * cm), 128: int(8 * cm), 256: int(4 * cm)}
    plog = int(math.ceil(math.log(opt.patch_size, 2)))
    ch = pch[2 ** plog]
    convlayer("Dpatch.convs.0", 3, ch, 3)
    for i in range(plog, 2, -1):
        nxt = pch[2 ** (i - 1)]
        name = str(7 - i) if i <= 6 else "%dx%d" % (2 ** i, 2 ** i)
        resblock("Dpatch.convs." + name, ch, nxt)
        ch = nxt
    resblock("Dpatch.convs.5", ch, cap * 2)
    convlayer("Dpatch.convs.6", cap * 2, cap, 3)
    for i, (a, b_) in enumerate([(pch[4] * 8, 2048), (2048, 2048), (2048, 1024), (1024, 1)]):
        lin("Dpatch.pairlinear.%d" % i, a, b_)
    return sd
