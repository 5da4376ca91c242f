"""fp32 CPU stand-ins for the `_lib` entry points the GatedPixelCNN, PixelSNAIL, VAE, VQ-VAE and VQ-VAE-2 stacks reach
(models/gated_pixel_cnn.py, models/pixel_snail.py, models/vae.py, models/vq_vae.py, models/vq_vae_2.py, nn/pm.py,
nn/modules.py, nn/vq.py), so that the product's own wiring runs without a GPU.  The direct image convolution and the
causal attention (strict included) are tests/_block_emulation.py's.  Shared by tests/test_conv_stack_bounds_cpu.py;
not a test module.

Each stand-in follows the rounding points of the C ABI (include/pg_b200.h), not its kernel's summation order: GEMM
operands are bf16 and every sum is fp32, split-K launches sum their slices in slice order, epilogues round to bf16 where
the kernel stores bf16, a gathered operand holds the bf16 values it was gathered from, pg_tap_scatter and
pg_strided_scatter add their taps in ascending tap order in fp32, the latent, quantizer and gate kernels round every
operation to fp32.  The bounds of tests/_conv_stack_reference.py hold for any fp32 summation order within the split-K
plan of the launch, so they must accept these stand-ins as they accept the kernels."""

import torch

import _block_emulation as BE
from _gemm_reference import split_plan

F32, BF16 = torch.float32, torch.bfloat16
ACT_NONE, ACT_RELU, ACT_ELU, ACT_TANH = 0, 1, 3, 4
ACT_GIVEN, ACT_RELU_OUT, ACT_ELU_OUT = 5, 6, 7
CONV_FWD, CONV_DGRAD, CONV_WGRAD = 1, 2, 3


def _act(t, act):
    act &= 0xFF
    if act == ACT_NONE:
        return t
    if act == ACT_RELU:
        return torch.relu(t)
    assert act == ACT_ELU, act
    return torch.nn.functional.elu(t)


def _dact(aux, dact):
    a = aux.float()
    if dact == ACT_GIVEN:
        return a
    if dact in (ACT_RELU, ACT_RELU_OUT):
        return (a > 0).float()
    assert dact == ACT_ELU_OUT, dact
    return torch.where(a > 0, torch.ones_like(a), a + 1)


def gemm(A, B, M, N, K, *, a_mn=False, b_mn=False, bias=None, aux=None, dact=ACT_NONE, res0=None, res1=None,
         out_bf16=None, out_pre=None, out_f32=None, act=ACT_NONE, accumulate=False, alpha=1.0, split_k=1, impl=0,
         bias_grad=None):
    assert A.dtype == BF16 and B.dtype == BF16
    a = (A.T if a_mn else A)[:M, :K].float()
    b = (B.T if b_mn else B)[:N, :K].float()
    _, kps, _ = split_plan(K, split_k)
    t = None
    for k0 in range(0, K, 64 * kps):  # one fp32 slice per split, added in slice order
        part = a[:, k0: k0 + 64 * kps] @ b[:, k0: k0 + 64 * kps].T
        t = part if t is None else t + part
    t = t * alpha
    if bias is not None:
        t = t + bias[:N]
    if dact != ACT_NONE:
        t = t * _dact(aux[:M, :N], dact)
    for r in (res0, res1):
        if r is not None:
            t = t + r[:M, :N].float()
    if out_f32 is not None:
        if accumulate:
            out_f32[:M, :N] += t
        else:
            out_f32[:M, :N] = t
    if out_bf16 is not None:
        out_bf16[:M, :N] = _act(t, act).to(BF16)
    if out_pre is not None:
        assert not act & 0x100
        out_pre[:M, :N] = t.to(BF16)
    if bias_grad is not None:
        bias_grad[:M] += a.sum(1)


def _shifted(x, N, H, W, C, taps, rows=None, stride=1):
    """[N * Hg * Wg, T * C] fp32: for every tap (dy, dx), x at (y s + dy, x s + dx), zero outside the image."""
    hg, wg = rows or (H, W)
    x4 = x[:, :C].float().reshape(N, H, W, C)
    m = max([abs(o) for t in taps for o in t] + [0]) + stride * max(hg, wg)
    xp = torch.zeros(N, H + 2 * m, W + 2 * m, C)
    xp[:, m: m + H, m: m + W] = x4
    cols = []
    for dy, dx in taps:
        v = xp[:, m + dy: m + dy + stride * hg: stride, m + dx: m + dx + stride * wg: stride]
        cols.append(v.reshape(N * hg * wg, C))
    return torch.cat(cols, 1)


def _fold(ycat, N, Hs, Ws, C, taps, rows=None, stride=1):
    """The adjoint of _shifted: fp32 [N * Hs * Ws, C], taps added in ascending order."""
    hg, wg = rows or (Hs, Ws)
    m = max([abs(o) for t in taps for o in t] + [0]) + stride * max(hg, wg)
    v = torch.zeros(N, Hs + 2 * m, Ws + 2 * m, C)
    for t, (dy, dx) in enumerate(taps):
        y = ycat[:, t * C:(t + 1) * C].float().reshape(N, hg, wg, C)
        v[:, m + dy: m + dy + stride * hg: stride, m + dx: m + dx + stride * wg: stride] += y
    return v[:, m: m + Hs, m: m + Ws].reshape(N * Hs * Ws, C)


def gemm_conv(A, B, M, N, K, mode, n_img, H, W, C, taps, *, bias=None, aux=None, dact=ACT_NONE, res0=None, res1=None,
              out_bf16=None, out_pre=None, out_f32=None, act=ACT_NONE, accumulate=False, alpha=1.0, split_k=1,
              bias_grad=None):
    kw = dict(bias=bias, aux=aux, dact=dact, res0=res0, res1=res1, out_bf16=out_bf16, out_pre=out_pre, out_f32=out_f32,
              act=act, accumulate=accumulate, alpha=alpha, split_k=split_k, bias_grad=bias_grad)
    T = len(taps)
    if mode == CONV_FWD:
        gemm(_shifted(A, n_img, H, W, C, taps).to(BF16), B, M, N, K, **kw)
    elif mode == CONV_DGRAD:  # B [Cout = C, T * N]: per tap W_t^T
        bt = B[:C, :T * N].reshape(C, T, N).permute(2, 1, 0).reshape(N, T * C)
        gemm(_shifted(A, n_img, H, W, C, taps).to(BF16), bt.contiguous(), M, N, K, **kw)
    else:
        assert mode == CONV_WGRAD
        gemm(A, _shifted(B, n_img, H, W, C, taps).to(BF16), M, N, K, a_mn=True, b_mn=True, **kw)


def tap_gather(x_pm, N, H, W, C, taps, act, out):
    out.copy_(_act(_shifted(x_pm, N, H, W, C, taps), act).to(BF16))


def tap_scatter(dxcat, N, H, W, C, taps, act, x_pre, dx_f32=None, dx_bf16=None):
    v = _fold(dxcat, N, H, W, C, taps)
    if act != ACT_NONE:
        v = v * _dact(x_pre[:, :C], act)
    if dx_f32 is not None:
        dx_f32[:, :C] = v
    if dx_bf16 is not None:
        dx_bf16[:, :C] = v.to(BF16)


def strided_gather(x_pm, rows, spatial, C, taps, stride, out):
    n, hs, ws = spatial
    out.copy_(_shifted(x_pm, n, hs, ws, C, taps, rows[1:], stride).to(BF16))


def strided_scatter(ycat, rows, spatial, C, taps, stride, *, bias=None, act=ACT_NONE, dact=ACT_NONE, x_pre=None,
                    out_f32=None, out_bf16=None):
    n, hs, ws = spatial
    v = _fold(ycat, n, hs, ws, C, taps, rows[1:], stride)
    if bias is not None:
        v[:, :bias.numel()] += bias
    if x_pre is not None:
        v = v * _dact(x_pre[:, :C], dact)
    if out_f32 is not None:
        out_f32[:, :C] = v
    if out_bf16 is not None:
        out_bf16[:, :C] = _act(v, act).to(BF16)


def act_cast(x, act, out):
    out.copy_(_act(x.float(), act).to(BF16))


def dact_from_out(dy, ya, act, out):
    out.copy_((dy.float() * _dact(ya, {ACT_ELU: ACT_ELU_OUT}.get(act, act))).to(BF16))


def _gate(x, act):
    c = x.shape[1] // 2
    f, g = x[:, :c].float(), x[:, c:].float()
    a = torch.tanh(f) if act == ACT_TANH else f
    return a, torch.sigmoid(g)


def gated_act_fwd(x, y, act):
    a, s = _gate(x, act)
    y.copy_((a * s).to(y.dtype))


def gated_act_bwd(x, dy, dx, act):
    a, s = _gate(x, act)
    d = dy.float()
    da = 1 - a * a if act == ACT_TANH else torch.ones_like(a)
    dx.copy_(torch.cat((d * s * da, d * a * s * (1 - s)), 1).to(dx.dtype))


def gated_res_fwd(x, res, y, act):
    a, s = _gate(x, act)
    y.copy_(res + a * s)


def vae_latent_fwd(h, eps, z, kl):
    n, L = eps.shape[:2]
    e = eps.permute(0, 2, 3, 1).reshape(-1, L)
    m, s = h[:, :L], h[:, L: 2 * L]
    z.zero_()
    z[:, :L] = (m + torch.exp(s) * e).to(BF16)
    t = -0.5 * (1 + 2 * s - torch.exp(s) ** 2 - m ** 2)
    kl.copy_(t.reshape(n, -1).sum(1))


def vae_latent_bwd(h, eps, dz, g_kl, dh):
    n, L = eps.shape[:2]
    e = eps.permute(0, 2, 3, 1).reshape(-1, L)
    m, s = h[:, :L], h[:, L: 2 * L]
    g = torch.zeros(h.shape[0], 1) if g_kl is None else g_kl.repeat_interleave(h.shape[0] // n)[:, None]
    d = dz[:, :L].float()
    dh.zero_()
    dh[:, :L] = (d + g * m).to(BF16)
    dh[:, L: 2 * L] = (d * torch.exp(s) * e + g * (torch.exp(s) ** 2 - 1)).to(BF16)


def vq_assign(x, emb, idx, out=None, col0=0, out_cols=None, loss_sum=None):
    d = emb.shape[1]
    xr = x[:, :d]
    dist = (xr * xr).sum(1, keepdim=True) + (emb * emb).sum(1) - 2 * xr @ emb.T
    i = torch.argmin(dist, 1)
    idx.copy_(i)
    q = emb[i]
    if out is not None:
        out[:, col0: col0 + d] = (xr + (q - xr)).to(out.dtype)
        out[:, col0 + d: col0 + (d if out_cols is None else out_cols)] = 0
    if loss_sum is not None:
        loss_sum += ((xr - q) ** 2).sum()


def vq_code_sums(x, idx, K, sums, counts=None, emb=None, g=None, scale=0.0):
    d = sums.shape[1]
    i = idx.long()
    rows = x[:, :d] if emb is None else ((emb[i] - x[:, :d]) * scale) * g[0]
    sums.zero_()
    sums.index_add_(0, i, rows)
    if counts is not None:
        counts.copy_(torch.bincount(i, minlength=K).float())


def vq_ema_update(counts, sums, decay, cluster_size, embedding_avg, embedding):
    cluster_size.mul_(decay).add_(counts * (1 - decay))
    embedding_avg.mul_(decay).add_(sums * (1 - decay))
    embedding.copy_(embedding_avg / (cluster_size + 1e-5)[:, None])


def vq_bwd(x, emb, idx, dq, col0, g, scale, dx):
    d = emb.shape[1]
    t = torch.zeros(x.shape[0], d) if dq is None else dq[:, col0: col0 + d].float()
    if g is not None:
        t = t + ((x[:, :d] - emb[idx.long()]) * scale) * g[0]
    dx.zero_()
    dx[:, :d] = t.to(dx.dtype)


def mse_mean(a, b, cols, *, loss_sum=None, g=None, scale=0.0, da=None, db=None):
    diff = a[:, :cols] - b[:, :cols]
    if loss_sum is not None:
        loss_sum += (diff ** 2).sum()
    if g is not None:
        t = (diff * scale) * g[0]
        for out, sign in ((da, 1), (db, -1)):
            if out is not None:
                out.zero_()
                out[:, :cols] = sign * t


STAND_INS = dict(gemm=gemm, gemm_conv=gemm_conv, tap_gather=tap_gather, tap_scatter=tap_scatter,
                 strided_gather=strided_gather, strided_scatter=strided_scatter, act_cast=act_cast,
                 dact_from_out=dact_from_out, vae_latent_fwd=vae_latent_fwd, vae_latent_bwd=vae_latent_bwd,
                 vq_assign=vq_assign, vq_code_sums=vq_code_sums, vq_ema_update=vq_ema_update, vq_bwd=vq_bwd,
                 mse_mean=mse_mean, gated_act_fwd=gated_act_fwd, gated_act_bwd=gated_act_bwd,
                 gated_res_fwd=gated_res_fwd,
                 causal_attn_fwd=BE.causal_attn_fwd, causal_attn_bwd=BE.causal_attn_bwd,
                 conv_small_fwd=BE.conv_small_fwd, conv_small_bwd=BE.conv_small_bwd,
                 colsum=BE.colsum, nchw_to_pm=BE.nchw_to_pm, pm_to_nchw=BE.pm_to_nchw,
                 cast_bf16=BE.cast_bf16, sm_count=BE.sm_count)


def install(monkeypatch):
    """Replaces the `_lib` entry points with the stand-ins, and lets the models' CUDA-only checks pass CPU tensors, for
    the rest of the test."""
    from pytorch_generative_b200 import _lib, losses
    from pytorch_generative_b200.models import vae, vq_vae, vq_vae_2
    from pytorch_generative_b200.nn import vq

    for name, fn in STAND_INS.items():
        monkeypatch.setattr(_lib, name, fn)
    for mod in (vae, vq_vae, vq_vae_2):
        monkeypatch.setattr(mod, "_require", lambda *a: None)
    monkeypatch.setattr(vq.VectorQuantizer, "_check", lambda self, z: None)
    monkeypatch.setattr(losses, "_mse_operand", lambda t, who: t.contiguous())
