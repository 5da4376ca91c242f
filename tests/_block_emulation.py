"""fp32 CPU stand-ins for the `_lib` entry points ImageGPT's fused stack reaches (models/image_gpt.py), so that the
product's own wiring (`_ImageGPTStack`, `_block_fwd`, `_block_bwd`, `GradArena`, the weight packing) runs without a GPU.
Shared by tests/test_block_bounds_cpu.py; not a test module.

Each stand-in follows the rounding points of the C ABI (include/pg_b200.h), not its kernel's summation order: GEMM
operands are bf16 and every sum is fp32, split-K launches sum their slices in slice order, GEMM epilogues round to bf16
where the kernel stores bf16, the attention kernels round P (forward and backward) and dS to bf16 before they multiply
them, and LayerNorm, the column sums and the input convolution run in fp32.  The bounds of tests/_block_reference.py
hold for any fp32 summation order, so they must accept these stand-ins as they accept the kernels.  Activations use the
exact erf GELU and its derivative, which are inside the kernels' documented fit error."""

import math

import torch

from _gemm_reference import split_plan

F32, BF16 = torch.float32, torch.bfloat16
ACT_NONE, ACT_GELU, ACT_GIVEN = 0, 2, 5
ACT_STORE_DERIV, ACT_RES_BF16 = 0x100, 0x200


def _gelu(x):
    return torch.nn.functional.gelu(x)


def _dgelu(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gemm(A, B, M, N, K, *, a_mn=False, b_mn=False, bias=None, aux=None, dact=ACT_NONE, res0=None, res1=None,
         out_bf16=None, out_pre=None, out_f32=None, act=ACT_NONE, accumulate=False, alpha=1.0, split_k=1, impl=0,
         bias_grad=None):
    assert A.dtype == BF16 and B.dtype == BF16
    a = (A.T if a_mn else A)[:M, :K].float()
    b = (B.T if b_mn else B)[:N, :K].float()
    _, kps, _ = split_plan(K, split_k)
    step = 64 * kps
    acc = None
    for k0 in range(0, K, step):  # one fp32 slice per split, added in slice order
        part = a[:, k0: k0 + step] @ b[:, k0: k0 + step].T
        acc = part if acc is None else acc + part
    t = acc * alpha
    if bias is not None:
        t = t + bias[:N]
    if dact != ACT_NONE:
        assert dact == ACT_GIVEN, dact
        t = t * aux[:M, :N].float()
    for r in (res0, res1):
        if r is not None:
            t = t + r[:M, :N].float()
    base = act & 0xFF
    assert base in (ACT_NONE, ACT_GELU), act
    if out_f32 is not None:
        if accumulate:
            out_f32[:M, :N] += t
        else:
            out_f32[:M, :N] = t
    if out_bf16 is not None:
        out_bf16[:M, :N] = (_gelu(t) if base == ACT_GELU else t).to(BF16)
    if out_pre is not None:
        out_pre[:M, :N] = (_dgelu(t) if act & ACT_STORE_DERIV else t).to(BF16)
    if bias_grad is not None:
        bias_grad[:M] += a.sum(1)


def colsum(x, out, accumulate=False):
    C = x.shape[1]
    s = x.float().sum(0)
    out[:C] = out[:C] + s if accumulate else s


def layernorm_fwd(x, gamma, beta, eps, y_bf16=None, y_f32=None, mean=None, rstd=None):
    C = gamma.numel()
    xc = x[:, :C]
    m = xc.sum(1, keepdim=True) / C
    var = ((xc - m) ** 2).sum(1, keepdim=True) / C
    r = torch.rsqrt(var + eps)
    y = torch.zeros_like(x)
    y[:, :C] = (xc - m) * r * gamma + beta
    if y_bf16 is not None:
        y_bf16.copy_(y.to(BF16))
    if y_f32 is not None:
        y_f32.copy_(y)
    mean.copy_(m[:, 0])
    rstd.copy_(r[:, 0])


def layernorm_bwd(dy, x, gamma, mean, rstd, dres0=None, dres1=None, dx_f32=None, dx_bf16=None, dgamma=None,
                  dbeta=None, dx_colsum=None):
    C = gamma.numel()
    g = dy[:, :C].float()
    xh = (x[:, :C] - mean[:, None]) * rstd[:, None]
    gy = g * gamma
    m1 = gy.sum(1, keepdim=True) / C
    m2 = (gy * xh).sum(1, keepdim=True) / C
    dx = rstd[:, None] * (gy - m1 - xh * m2)
    for r in (dres0, dres1):
        if r is not None:
            dx = dx + r[:, :C]
    full = torch.zeros(x.shape, dtype=F32)
    full[:, :C] = dx
    if dx_f32 is not None:
        dx_f32.copy_(full)
    if dx_bf16 is not None:
        dx_bf16.copy_(full.to(BF16))
    if dgamma is not None:
        dgamma += (g * xh).sum(0)
    if dbeta is not None:
        dbeta += g.sum(0)
    if dx_colsum is not None:
        dx_colsum += dx.sum(0)


def nchw_to_pm(x, out):
    n, c, h, w = x.shape
    out.copy_(x.permute(0, 2, 3, 1).reshape(n * h * w, c).to(out.dtype))


def pm_to_nchw(x_pm, out, act=ACT_NONE):
    assert act == ACT_NONE
    n, c, h, w = out.shape
    out.copy_(x_pm.float().reshape(n, h, w, c).permute(0, 3, 1, 2))


def cast_bf16(x, y):
    y.copy_(x.to(BF16))


def _heads(t, N, S, H, d):
    """[N S, H d] pixel-major head slots -> fp32 [N, H, S, d]."""
    return t[:, : H * d].float().reshape(N, S, H, d).permute(0, 2, 1, 3)


def _store(t, out, N, S, H, d):
    out.copy_(t.permute(0, 2, 1, 3).reshape(N * S, H * d).to(out.dtype))


def _scores(q, k, N, S, H, dk, scale, strict=False):
    """Scores with the keys j <= i visible (j < i when strict); a strict row 0 sees none and is all -inf."""
    s = (_heads(q, N, S, H, dk) @ _heads(k, N, S, H, dk).transpose(-1, -2)) * scale
    vis = torch.tril(torch.ones(S, S, dtype=torch.bool), diagonal=-int(strict))
    return s.masked_fill(~vis, -math.inf)


def causal_attn_fwd(q, k, v, o, lse, N, S, H, dk, dv, strict, impl=0, dk_true=None):
    """A row without visible keys (strict row 0) gets o = 0 and lse = 0, as the kernels define it."""
    s = _scores(q, k, N, S, H, dk, 1.0 / math.sqrt(dk_true or dk), strict)
    m = s.amax(-1, keepdim=True)
    none = torch.isinf(m)
    m = m.masked_fill(none, 0.0)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    _store(((e.to(BF16).float() @ _heads(v, N, S, H, dv)) / l.masked_fill(none, 1.0)).masked_fill(none, 0.0), o, N, S,
           H, dv)
    lse.copy_((m + torch.log(l.masked_fill(none, 1.0)))[..., 0])


def causal_attn_bwd(q, k, v, o, do, lse, delta, dq_accum, dq, dk_, dv_, N, S, H, dk, dv, strict, impl=0, dk_true=None):
    c = 1.0 / math.sqrt(dk_true or dk)
    p = torch.exp(_scores(q, k, N, S, H, dk, c, strict) - lse[..., None])
    dO, V = _heads(do, N, S, H, dv), _heads(v, N, S, H, dv)
    D = (dO * _heads(o, N, S, H, dv)).sum(-1, keepdim=True)
    delta.copy_(D[..., 0])
    dS = (p * (dO @ V.transpose(-1, -2) - D)).to(BF16).float()
    _store(p.to(BF16).float().transpose(-1, -2) @ dO, dv_, N, S, H, dv)
    _store(c * (dS @ _heads(k, N, S, H, dk)), dq, N, S, H, dk)
    _store(c * (dS.transpose(-1, -2) @ _heads(q, N, S, H, dk)), dk_, N, S, H, dk)


def conv_small_fwd(x, w, bias, pad, out_f32=None, out_bf16=None, act_bf16=ACT_NONE, pre_act=ACT_NONE, dilation=(1, 1)):
    """The front crop to x's H x W of the padded convolution, like the kernel."""
    assert pre_act == ACT_NONE and act_bf16 == ACT_NONE and out_bf16 is None and tuple(dilation) == (1, 1)
    n, _, h, wd = x.shape
    y = torch.nn.functional.conv2d(x, w, bias, padding=tuple(pad))[:, :, :h, :wd]
    out_f32.copy_(y.permute(0, 2, 3, 1).reshape(-1, w.shape[0]))


def conv_small_bwd(x, w, dy_pm, pad, dw=None, dbias=None, dx=None, pre_act=ACT_NONE, dilation=(1, 1)):
    assert pre_act == ACT_NONE and tuple(dilation) == (1, 1)
    n, _, h, wd = x.shape
    kh, kw = w.shape[-2:]
    dy = torch.zeros(n, w.shape[0], h + 2 * pad[0] - kh + 1, wd + 2 * pad[1] - kw + 1)  # the cropped-off rows get none
    dy[:, :, :h, :wd] = dy_pm.reshape(n, h, wd, w.shape[0]).permute(0, 3, 1, 2)
    if dw is not None:
        dw += torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=tuple(pad))
    if dbias is not None:
        dbias += dy.sum((0, 2, 3))
    if dx is not None:
        dx.copy_(torch.nn.grad.conv2d_input(x.shape, w, dy, padding=tuple(pad)))


def sm_count():
    return 132


def cast_multi(*args, **kwargs):
    raise NotImplementedError("cast_multi packs through raw device pointers: the slot-filling packing needs the GPU")


STAND_INS = dict(gemm=gemm, colsum=colsum, layernorm_fwd=layernorm_fwd, layernorm_bwd=layernorm_bwd,
                 nchw_to_pm=nchw_to_pm, pm_to_nchw=pm_to_nchw, cast_bf16=cast_bf16, causal_attn_fwd=causal_attn_fwd,
                 causal_attn_bwd=causal_attn_bwd, conv_small_fwd=conv_small_fwd, conv_small_bwd=conv_small_bwd,
                 sm_count=sm_count, cast_multi=cast_multi)


def install(monkeypatch):
    """Replaces the `_lib` entry points with the stand-ins for the rest of the test."""
    from pytorch_generative_b200 import _lib

    for name, fn in STAND_INS.items():
        monkeypatch.setattr(_lib, name, fn)
