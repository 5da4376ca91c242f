"""Convolutions of any kernel size up to 15 x 15 (225 taps) and any dilation, on the GPU.

Kernels against float64, element by element, in the style of tests/_gemm_reference.py: inputs are rounded to bf16 first,
every product of two bf16 values is exact in fp32, and a sum of n terms rounded to fp32 is within (n - 1) U24 sum|terms|
of the exact sum whatever the order, so
  * the tap-loop GEMM forward and dgrad (K = T C products, then the bias / output rounding) are held to
    (T C + 3) U24 times the tap sum of absolute values, and its wgrad (K = pixels, split along pixels) to
    (P + 2) U24 sum_p |dy| |x|, like test_conv_path_kernels_gpu.py's tap-loop cases;
  * tap gather is a copy: bit for bit;
  * tap scatter adds at most T bf16 terms in fp32: (T + 2) U24 sum_t |terms|.
Every operand and output is a view into a NaN-filled buffer (pitch wider than the view), so a read or a write outside
the view shows up, and every launch runs twice: identical bits.

Modules against torch.nn.functional.conv2d on the masked weight (the reference's CausalConv2d): the output, the input
gradient, the dense weight gradient (masked positions included) and the bias gradient, within 1e-2 on the bf16 path and
1e-3 on the fp32 direct kernel of image-channel layers.  Models against the oracle: PixelCNN with four image channels and
with 192 residual channels (input layers the direct kernel cannot take), a FusedAdam trajectory, and teacher-forced
incremental sampling at four image channels.  Outputs and logits are held to tol * max(1, max|ref|).  Every gradient is
held to a bound relative to its own max|ref|, with no floor, and the cotangents are unscaled randn, so a gradient that
a bug zeroed fails: tol for the modules, and for the models a per-parameter budget derived from the oracle itself
(`_rounding_budget`)."""

import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24
F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
TOL_BF16, TOL_F32 = 1e-2, 1e-3
GAMMA = 0.999977


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _dev():
    return torch.device("cuda:0")


def _randn(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(_dev())


def _view(P, C, dtype, extra=24, fill=float("nan")):
    """[P, C] view (unit inner stride, pitch C + extra) of a buffer filled with `fill`; returns (view, buffer)."""
    buf = torch.full((P, C + extra), fill, dtype=dtype, device=_dev())
    return buf[:, :C], buf


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def check(name, got, ref, a):
    """|got - ref| <= a element by element; NaN fails.  Names the worst element."""
    g, ref = got.to(F64), ref.to(F64)
    err = (g - ref).abs()
    bad = ~(err <= a)
    if bad.any():
        ratio = torch.where(bad, (err / a).nan_to_num(nan=math.inf, posinf=math.inf), torch.zeros_like(err))
        idx = tuple(int(i) for i in torch.unravel_index(ratio.reshape(-1).argmax().cpu(), g.shape))
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound; worst at {idx}: "
                             f"got {g[idx].item()!r}, ref {ref[idx].item()!r}, bound {a[idx].item():.3e}")


def check_equal(name, got, ref):
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape)
    bad = _bits(got) != _bits(ref)
    assert not bad.any(), f"{name}: {int(bad.sum())}/{bad.numel()} elements differ"


def check_untouched(name, buf, C):
    assert bool(buf[:, C:].isnan().all()), f"{name}: wrote past column {C}"


def _shift(x, dy, dx):
    """out[n, h, w] = x[n, h + dy, w + dx], zero outside the image (x: [N, H, W, C])."""
    N, H, W, C = x.shape
    out = torch.zeros_like(x)
    h0, h1 = max(0, -dy), min(H, H - dy)
    w0, w1 = max(0, -dx), min(W, W - dx)
    if h1 > h0 and w1 > w0:
        out[:, h0:h1, w0:w1] = x[:, h0 + dy:h1 + dy, w0 + dx:w1 + dx]
    return out


def _tap_sum(x_pm, w_cat, geom, taps, sign=1):
    """sum_t shift(x, sign * off_t) @ W_t^T with W_t = w_cat[:, t C:(t + 1) C] (float64, [P, Cout])."""
    n, h, w = geom
    C = x_pm.shape[1]
    x4 = x_pm.reshape(n, h, w, C)
    out = 0
    for t, (a, b) in enumerate(taps):
        out = out + _shift(x4, sign * a, sign * b).reshape(-1, C) @ w_cat[:, t * C:(t + 1) * C].t()
    return out


def _tap_sum_t(dy64, w64, geom, taps):
    """Dgrad of the tap sum: dx[p] = sum_t W_t^T dy[p - off_t] (float64, [P, Cin])."""
    n, h, w = geom
    Cout = dy64.shape[1]
    Cin = w64.shape[1] // len(taps)
    d4 = dy64.reshape(n, h, w, Cout)
    out = 0
    for t, (a, b) in enumerate(taps):
        out = out + _shift(d4, -a, -b).reshape(-1, Cout) @ w64[:, t * Cin:(t + 1) * Cin]
    return out


# ----------------------------------------------------------------------------------------------------------------------
# A. tap-loop GEMM (pg_gemm_bf16_conv_taps)
# ----------------------------------------------------------------------------------------------------------------------
# name: (N, H, W, Cin, Cout, (kh, kw), dilation).  Padding d (k // 2): 'same' offsets (i d - pad); every case has taps
# that reach past the image's edge rows and columns.  Cout = 72 and 200 leave partial N tiles.
TAP_LOOP_CASES = {
    "T33_3x11_d12": (2, 16, 16, 64, 72, (3, 11), (1, 2)),
    "T49_7x7_d1": (2, 16, 8, 128, 64, (7, 7), (1, 1)),
    "T81_9x9_d2": (1, 32, 32, 64, 200, (9, 9), (2, 2)),
    "T81_9x9_d3": (1, 16, 64, 64, 128, (9, 9), (3, 3)),
    "T225_15x15_d1": (1, 16, 32, 64, 64, (15, 15), (1, 1)),
    "T225_15x15_d3": (1, 32, 64, 64, 128, (15, 15), (3, 3)),
}


@pytest.mark.parametrize("case", list(TAP_LOOP_CASES))
def test_tap_loop_gemm_many_taps(L, case):
    from pytorch_generative_b200 import ops
    from pytorch_generative_b200.nn.tapconv import conv_taps

    N, H, W, Cin, Cout, (kh, kw), (dh, dw) = TAP_LOOP_CASES[case]
    taps = conv_taps(kh, kw, dh * (kh // 2), dw * (kw // 2), dh, dw)
    T, P, geom = len(taps), N * H * W, (N, H, W)
    assert T == kh * kw and L.conv_gemm_supported(H, W, Cin, taps)
    seed = 1000 + T
    x, _ = _view(P, Cin, BF16)
    x.copy_(_randn((P, Cin), seed).to(BF16))
    wcat, _ = _view(Cout, T * Cin, BF16)
    wcat.copy_(_randn((Cout, T * Cin), seed + 1, 2 / math.sqrt(T * Cin)).to(BF16))
    bias = _randn((Cout,), seed + 2)
    x64, w64 = x.to(F64), wcat.to(F64)

    # forward: y = bias + sum_t W_t x[p + off_t]
    runs = []
    for _ in range(2):
        yf, yf_buf = _view(P, Cout, F32)
        yb, yb_buf = _view(P, Cout, BF16)
        L.gemm_conv(x, wcat, P, Cout, T * Cin, L.CONV_FWD, N, H, W, Cin, taps, bias=bias, out_f32=yf, out_bf16=yb)
        runs.append((yf, yf_buf, yb, yb_buf))
    torch.cuda.synchronize()
    yf, yf_buf, yb, yb_buf = runs[0]
    ref = _tap_sum(x64, w64, geom, taps) + bias.to(F64)
    mag = _tap_sum(x64.abs(), w64.abs(), geom, taps) + bias.to(F64).abs()
    check(f"{case}: fwd out_f32", yf, ref, (T * Cin + 3) * U24 * mag)
    check_equal(f"{case}: fwd out_bf16 = bf16(out_f32)", yb, yf.to(BF16))
    check_untouched(f"{case}: fwd out_f32", yf_buf, Cout)
    check_untouched(f"{case}: fwd out_bf16", yb_buf, Cout)
    check_equal(f"{case}: fwd repeated", runs[1][0], yf)

    # dgrad: dx = sum_t W_t^T dy[p - off_t] (the shifted operand is dy: Cout % 64)
    if Cout % 64 == 0:
        dy, _ = _view(P, Cout, BF16)
        dy.copy_(_randn((P, Cout), seed + 3).to(BF16))
        runs = []
        for _ in range(2):
            dx, dx_buf = _view(P, Cin, F32)
            L.gemm_conv(dy, wcat, P, Cin, T * Cout, L.CONV_DGRAD, N, H, W, Cout, [(-a, -b) for a, b in taps], out_f32=dx)
            runs.append((dx, dx_buf))
        torch.cuda.synchronize()
        dx, dx_buf = runs[0]
        dy64 = dy.to(F64)
        check(f"{case}: dgrad", dx, _tap_sum_t(dy64, w64, geom, taps),
              (T * Cout + 3) * U24 * _tap_sum_t(dy64.abs(), w64.abs(), geom, taps))
        check_untouched(f"{case}: dgrad", dx_buf, Cin)
        check_equal(f"{case}: dgrad repeated", runs[1][0], dx)

    # wgrad: dW[:, t C + c] += sum_p dy[p] x[p + off_t, c], the bias gradient on the same launch
    dy, _ = _view(P, Cout, BF16)
    dy.copy_(_randn((P, Cout), seed + 4).to(BF16))
    runs = []
    for _ in range(2):
        dW, dW_buf = _view(Cout, T * Cin, F32)
        dW.zero_()
        db = torch.full((Cout,), 0.5, device=_dev())
        ops.conv_wgrad(dy, x, dW, N, H, W, taps, db_out=db)
        runs.append((dW, dW_buf, db))
    torch.cuda.synchronize()
    dW, dW_buf, db = runs[0]
    dy64 = dy.to(F64)
    x4 = x64.reshape(N, H, W, Cin)
    xs = torch.cat([_shift(x4, a, b).reshape(P, Cin) for a, b in taps], dim=1)
    check(f"{case}: wgrad", dW, dy64.t() @ xs, (P + 2) * U24 * (dy64.abs().t() @ xs.abs()))
    check(f"{case}: wgrad bias gradient", db, dy64.sum(0) + 0.5, (P + 2) * U24 * (dy64.abs().sum(0) + 0.5))
    check_untouched(f"{case}: wgrad", dW_buf, T * Cin)
    check_equal(f"{case}: wgrad repeated", runs[1][0], dW)
    check_equal(f"{case}: bias gradient repeated", runs[1][2], db)


def test_tap_loop_refuses_offsets_beyond_64(L):
    x = torch.zeros(128, 64, dtype=BF16, device=_dev())
    w = torch.zeros(64, 2 * 64, dtype=BF16, device=_dev())
    y = torch.zeros(128, 64, device=_dev())
    with pytest.raises(RuntimeError, match="tap offset out of range"):
        L.gemm_conv(x, w, 128, 64, 128, L.CONV_FWD, 1, 16, 8, 64, [(0, 0), (-65, 0)], out_f32=y)


# ----------------------------------------------------------------------------------------------------------------------
# B. tap gather / scatter
# ----------------------------------------------------------------------------------------------------------------------
# name: (N, H, W, C, (kh, kw), dilation, padding)
GATHER_CASES = {
    "T33_3x11_d12": (2, 12, 20, 8, (3, 11), (1, 2), (1, 10)),
    "T49_7x7_d1": (2, 28, 28, 136, (7, 7), (1, 1), (3, 3)),
    "T81_9x9_d3": (1, 30, 26, 16, (9, 9), (3, 3), (12, 12)),
    "T225_15x15_d2": (1, 20, 24, 24, (15, 15), (2, 2), (14, 14)),
    "T9_3x3_d70": (1, 150, 9, 16, (3, 3), (70, 1), (70, 1)),        # dy = +-70: beyond the tap loop's 64
    "T225_15x15_d5": (1, 80, 72, 8, (15, 15), (5, 5), (35, 35)),    # dy, dx up to 35 on a 80 x 72 image
}


def _gather_taps(case):
    from pytorch_generative_b200.nn.tapconv import conv_taps

    n, h, w, C, (kh, kw), (dh, dw), (ph, pw) = GATHER_CASES[case]
    return (n, h, w, C), conv_taps(kh, kw, ph, pw, dh, dw)


@pytest.mark.parametrize("case", list(GATHER_CASES))
def test_tap_gather_many_taps(L, case):
    """X_cat[p, t C + c] = x[p + off_t, c] (zero outside the image), and relu of it: copies, bit for bit."""
    (n, h, w, C), taps = _gather_taps(case)
    T, P = len(taps), n * h * w
    x, _ = _view(P, C, BF16, extra=8)
    x.copy_(_randn((P, C), 2000 + T).to(BF16))
    x4 = x.to(F64).reshape(n, h, w, C)
    for act in (L.ACT_NONE, L.ACT_RELU):
        src = x4 if act == L.ACT_NONE else x4.clamp_min(0)
        ref = torch.cat([_shift(src, a, b).reshape(P, C) for a, b in taps], dim=1).to(BF16)
        outs = []
        for _ in range(2):  # X_cat is dense [P, T C]: a NaN tail after it shows a write past its end
            buf = torch.full((P * T * C + 64,), float("nan"), dtype=BF16, device=_dev())
            L.tap_gather(x, n, h, w, C, taps, act, buf[:P * T * C].view(P, T * C))
            outs.append(buf)
        torch.cuda.synchronize()
        check_equal(f"{case} act {act}: gather", outs[0][:P * T * C].view(P, T * C), ref)
        assert bool(outs[0][P * T * C:].isnan().all()), f"{case}: gather wrote past X_cat"
        check_equal(f"{case} act {act}: gather repeated", outs[1], outs[0])


@pytest.mark.parametrize("case", list(GATHER_CASES))
def test_tap_scatter_many_taps(L, case):
    """dx[p, c] = act'(x_pre[p, c]) sum_t dX_cat[p - off_t, t C + c] into pitched fp32 and bf16 views: at most T fp32
    additions of bf16 terms, then the derivative (0 or 1 for ReLU, exact): (T + 2) U24 sum_t |terms| |g|."""
    (n, h, w, C), taps = _gather_taps(case)
    T, P = len(taps), n * h * w
    dxcat = _randn((P, T * C), 3000 + T).to(BF16)
    x_pre, _ = _view(P, C, BF16, extra=8)
    x_pre.copy_(_randn((P, C), 3001 + T).to(BF16))

    def scattered(d):
        return sum(_shift(d[:, t * C:(t + 1) * C].reshape(n, h, w, C), -a, -b).reshape(P, C)
                   for t, (a, b) in enumerate(taps))

    s, s_abs = scattered(dxcat.to(F64)), scattered(dxcat.to(F64).abs())
    for act in (L.ACT_NONE, L.ACT_RELU):
        g = torch.ones_like(s) if act == L.ACT_NONE else (x_pre.to(F64) > 0).to(F64)
        runs = []
        for _ in range(2):
            buf_f = torch.full((P, C + 8), float("nan"), device=_dev())
            buf_b = torch.full((P, C + 8), float("nan"), dtype=BF16, device=_dev())
            L.tap_scatter(dxcat, n, h, w, C, taps, act, x_pre, dx_f32=buf_f[:, :C], dx_bf16=buf_b[:, :C])
            runs.append((buf_f, buf_b))
        torch.cuda.synchronize()
        (buf_f, buf_b), (buf_f2, _) = runs
        check(f"{case} act {act}: scatter dx_f32", buf_f[:, :C], s * g, (T + 2) * U24 * s_abs * g)
        check_equal(f"{case} act {act}: dx_bf16 = bf16(dx_f32)", buf_b[:, :C], buf_f[:, :C].to(BF16))
        check_untouched(f"{case} act {act}: dx_f32", buf_f, C)
        check_untouched(f"{case} act {act}: dx_bf16", buf_b, C)
        check_equal(f"{case} act {act}: scatter repeated", buf_f2, buf_f)


# ----------------------------------------------------------------------------------------------------------------------
# C. CausalConv2d against F.conv2d on the masked weight
# ----------------------------------------------------------------------------------------------------------------------
def relcheck(name, got, ref, tol, floor=1.0):
    """max |got - ref| <= tol * max(floor, max|ref|).  floor = 0 holds a gradient to its own scale; its reference must
    then be nonzero, so that a result of all zeros fails."""
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    scale = max(floor, ref.abs().max().item())
    assert scale > 0, f"{name}: the reference is zero, so the check could not fail"
    bound = tol * scale
    err = (got - ref).abs().max().item()
    assert err <= bound and not torch.isnan(got).any(), f"{name}: max err {err:.3e} > {bound:.3e} (max|ref| {scale:.3e})"


def gradcheck(name, got, ref, tol):
    relcheck(name, got, ref, tol, floor=0.0)


def _spy(monkeypatch):
    """Counts the tap-loop GEMM and tap-gather launches of the module under test."""
    from pytorch_generative_b200 import _lib

    seen = {"gemm_conv": 0, "tap_gather": 0}
    for name in seen:
        real = getattr(_lib, name)

        def wrapped(*a, _real=real, _name=name, **k):
            seen[_name] += 1
            return _real(*a, **k)

        monkeypatch.setattr(_lib, name, wrapped)
    return seen


def _module_case(monkeypatch, mask_center, cin, cout, k, dilation, shape, tol, seed=0):
    """CausalConv2d(mask_center, cin, cout, k, padding=d (k // 2), dilation=d) against float64 F.conv2d on the masked
    weight: output and a fixed-cotangent VJP for the input, the dense weight gradient and the bias.  Returns the launch
    counts of the two wide-channel paths."""
    from pytorch_generative_b200 import nn

    kh, kw = (k, k) if isinstance(k, int) else k
    dh, dw = (dilation, dilation) if isinstance(dilation, int) else dilation
    torch.manual_seed(seed)
    m = nn.CausalConv2d(mask_center, cin, cout, (kh, kw), padding=(dh * (kh // 2), dw * (kw // 2)), dilation=(dh, dw))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        m.weight.mul_(4.0)   # outputs of order one: the tolerance is relative to max(1, max|ref|)
    x = torch.randn(shape, generator=g)
    n, _, h, w = shape
    G = torch.randn(n, cout, h, w, generator=g)

    wm = (m.weight.detach() * m.mask).double().requires_grad_(True)
    b = m.bias.detach().double().requires_grad_(True)
    xr = x.double().requires_grad_(True)
    ref = F.conv2d(xr, wm, b, padding=m.padding, dilation=m.dilation)[:, :, :h, :w]
    (ref * G.double()).sum().backward()

    seen = _spy(monkeypatch)
    m = m.to(_dev())
    xd = x.to(_dev()).requires_grad_(True)
    y = m(xd)
    (y * G.to(_dev())).sum().backward()
    torch.cuda.synchronize()
    tag = f"CausalConv2d({mask_center}, {cin}, {cout}, {(kh, kw)}, dilation={(dh, dw)}) on {tuple(shape)}"
    relcheck(f"{tag}: output", y, ref, tol)
    gradcheck(f"{tag}: input gradient", xd.grad, xr.grad, tol)
    gradcheck(f"{tag}: weight gradient (dense)", m.weight.grad, wm.grad, tol)
    gradcheck(f"{tag}: bias gradient", m.bias.grad, b.grad, tol)
    masked = (m.weight.grad * (1 - m.mask)).abs().sum().item()
    assert masked > 0, f"{tag}: the masked weight positions received no gradient"
    return seen


MODULE_KERNELS = {"7x7": (7, 1), "9x9": (9, 1), "3x5": ((3, 5), 1), "5x5_d2": (5, 2), "15x15": (15, 1),
                  "7x7_d2x1": (7, (2, 1))}


@pytest.mark.parametrize("shape", [(2, 32, 32), (2, 28, 28)], ids=["32x32", "28x28"])
@pytest.mark.parametrize("channels", [64, 100])
@pytest.mark.parametrize("mask_center", [True, False], ids=["A", "B"])
@pytest.mark.parametrize("kernel", list(MODULE_KERNELS))
def test_causal_conv2d_wide_channels(monkeypatch, kernel, mask_center, channels, shape):
    """The bf16 path: the TMA tap loop at 64 channels on 32 x 32 images, the gather path at 100 channels or 28 x 28."""
    k, d = MODULE_KERNELS[kernel]
    n, h, w = shape
    seen = _module_case(monkeypatch, mask_center, channels, channels, k, d, (n, channels, h, w), TOL_BF16)
    tap_loop = channels % 64 == 0 and w == 32
    assert (seen["gemm_conv"] > 0, seen["tap_gather"] > 0) == (tap_loop, not tap_loop), seen


def test_causal_conv2d_offsets_beyond_64_take_the_gather_path(monkeypatch):
    """64 channels on a 130 x 64 image suit the tap loop, but dilation 65 puts taps at dy = -65: gather."""
    seen = _module_case(monkeypatch, True, 64, 64, 3, 65, (1, 64, 130, 64), TOL_BF16)
    assert seen["gemm_conv"] == 0 and seen["tap_gather"] > 0, seen


@pytest.mark.parametrize("k,d,cin,cout", [(7, 1, 3, 32), (5, 2, 3, 16), (3, 3, 1, 16), ((3, 5), (2, 1), 3, 8),
                                          (7, 2, 1, 32)])
@pytest.mark.parametrize("mask_center", [True, False], ids=["A", "B"])
def test_causal_conv2d_image_channels_stay_fp32(monkeypatch, k, d, cin, cout, mask_center):
    """Image-channel layers, dilated ones included, run on the fp32 direct kernel: 1e-3."""
    seen = _module_case(monkeypatch, mask_center, cin, cout, k, d, (2, cin, 28, 28), TOL_F32)
    assert seen["gemm_conv"] == 0 and seen["tap_gather"] == 0, seen


# ----------------------------------------------------------------------------------------------------------------------
# D. PixelCNN against the oracle
# ----------------------------------------------------------------------------------------------------------------------
def _pcnn(c, res, n_res=2, head=16):
    return dict(in_channels=c, out_channels=c, n_residual=n_res, residual_channels=res, head_channels=head)


PCNN = {"c4_res16": _pcnn(4, 16), "c4_res64": _pcnn(4, 64), "c3_res192": _pcnn(3, 192, n_res=3, head=32)}


def _image(shape, g):
    return torch.randint(0, 256, shape, generator=g).float() / 255


def _perturbed(cfg, seed=0):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = models.PixelCNN(**cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=g) * 0.02)
    return m, g


def _rounding_budget(cfg, state, x, G, ref_grads):
    """Per-parameter gradient bounds relative to each gradient's own max|ref|: three times what rounding the oracle's
    conv weights and the image to bf16 does to that gradient (the CUDA path rounds them, and every activation, to bf16
    operands), never less than TOL_BF16.  A fixed 1 % does not hold for these models: ReLU gates flipped by rounding-sized
    changes move, e.g., the 7x7 input layer's weight gradient by 3-7 % of its max|ref| in the oracle itself.  The same
    rule as the ImageGPT bounds in test_channel_counts_gpu.py."""
    from oracle import reference_path as O

    rounded = {k: (v.to(BF16).float() if k.endswith("weight") else v) for k, v in state.items()}
    pt = O.trainable(rounded)
    (O.forward("pixel_cnn", pt, x.to(BF16).float(), cfg) * G).sum().backward()
    return {k: max(TOL_BF16, 3 * (pt[k].grad - r).abs().max().item() / r.abs().max().item()) for k, r in ref_grads.items()}


@pytest.mark.parametrize("size", [28, 32])
@pytest.mark.parametrize("key", sorted(PCNN))
def test_pixel_cnn_matches_oracle(key, size):
    """Logits and loss within 1e-2; every parameter's gradient within its rounding budget (`_rounding_budget`) of its own
    max|ref|.  Every budget stays below 1/2, so a gradient that is zero, or off by its own size, fails."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import losses, models, nn

    cfg = PCNN[key]
    assert not nn.tapconv.small_conv_ok(models.PixelCNN(**cfg)._input.weight.shape)  # the input layer takes the tap path
    m, g = _perturbed(cfg)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    c = cfg["in_channels"]
    x = _image((2, c, size, size), g)
    G = torch.randn(2, c, size, size, generator=g)
    pt = O.trainable(state)
    ref_logits = O.forward("pixel_cnn", pt, x, cfg)
    ref_loss = O.recipe_loss(x, ref_logits).detach()
    (ref_logits * G).sum().backward()
    ref_grads = {k: v.grad for k, v in pt.items() if v.grad is not None}
    tol = _rounding_budget(cfg, state, x, G, ref_grads)

    m = m.to(_dev())
    xd = x.to(_dev())
    logits = m(xd)
    loss = losses.bce_with_logits_sum_mean(logits, xd)
    (logits * G.to(_dev())).sum().backward()
    relcheck("logits", logits, ref_logits, TOL_BF16)
    assert abs(loss.item() - ref_loss.item()) <= TOL_BF16 * abs(ref_loss.item()), (loss.item(), ref_loss.item())
    report, ok = [], True
    for name, p in m.named_parameters():
        r = ref_grads[name]
        scale = r.abs().max().item()
        err = (p.grad.detach().float().cpu() - r).abs().max().item() / scale
        assert tol[name] < 0.5, f"d{name}: a budget of {tol[name]:.3f} of max|ref| could not see a wrong gradient"
        report.append(f"d{name:40s} max|ref| {scale:9.3e}  err/max|ref| {err:.3e}  budget {tol[name]:.3e}")
        ok &= err <= tol[name] and not p.grad.isnan().any().item()
    assert len(report) == len(ref_grads) == len(list(m.parameters()))
    print("\n".join(report))
    assert ok, "gradients:\n" + "\n".join(report)


def test_pixel_cnn_fused_adam_trajectory_matches_oracle():
    from oracle import reference_path as O
    from pytorch_generative_b200 import losses, optim

    cfg = PCNN["c4_res16"]
    lr = 1e-3
    m, g = _perturbed(cfg)
    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    xs = [_image((2, 4, 16, 16), g) for _ in range(3)]
    ts = O.TrainState("pixel_cnn", init, cfg, lr=lr, lr_gamma=GAMMA)
    ref = [ts.step(x) for x in xs]
    m = m.to(_dev()).train()
    opt = optim.FusedAdam(m.parameters(), lr=lr)
    sched = torch.optim.lr_scheduler.MultiplicativeLR(opt, lr_lambda=lambda _: GAMMA)
    for k, x in enumerate(xs):
        xd = x.to(_dev())
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(m(xd), xd)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(list(m.parameters()), 1e50)
        opt.step()
        sched.step()
        rl, rn = ref[k]
        assert abs(loss.item() - rl) <= TOL_BF16 * (1 + k) * abs(rl), (k, loss.item(), rl)
        assert abs(norm.item() - rn) <= 2.5e-2 * (1 + 1.5 * k) * abs(rn), (k, norm.item(), rn)
    worst = max(float((p.detach().cpu() - ts.p[n_].detach()).abs().max()) for n_, p in m.named_parameters())
    assert worst <= 2.0 * 3 * lr * 1.05


@pytest.mark.parametrize("shape", [(2, 4, 12, 20), (3, 4, 28, 28)], ids=["12x20", "28x28"])
def test_pixel_cnn_samples_four_channels_incrementally(shape):
    """Teacher-forced per-pixel logits of `sample()` (the 24 live taps of the 7x7 type-A mask) against the full
    forward, whose input layer runs on the tap path; two calls, the second replays the captured graph."""
    from pytorch_generative_b200 import models

    torch.manual_seed(7)
    m = models.PixelCNN(**_pcnn(4, 16)).to(_dev())
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.5)
    x = torch.bernoulli(torch.full(shape, 0.5)).to(_dev())
    with torch.no_grad():
        ref = m(x)
    n, c, h, w = shape
    assert m._incremental_ok(x)
    for rep in range(2):
        seen = []
        m._sample_fn = lambda logits: (seen.append(logits.detach().clone()), logits.new_zeros(n, c))[1]
        assert torch.equal(m.sample(conditioned_on=x), x)
        assert len(seen) == h * w
        relcheck(f"incremental logits (call {rep})", torch.stack(seen, dim=-1).view(ref.shape), ref, TOL_BF16)
    assert all(st["graph"] for st in m._pixel_states.values()), "per-pixel program was not graph-captured"
