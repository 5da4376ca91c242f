"""VeryDeepVAE on the GPU: every new kernel against float64 with per-element bounds, `pm.conv` with a GELU input in all
three modes, and the model against the reference fixture and the float64 restatement, with determinism, the FusedAdam
trajectory, the CUDA-graph step, sampling, the recipe and deepcopy / pickle."""

import copy
import os
import pickle
import sys

import pytest
import torch
from torch.nn import functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _vd_vae_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vd_vae.pt")
F64, BF16 = torch.float64, torch.bfloat16


def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def fixture():
    return R.load_fixture(GOLD)


@pytest.fixture
def recorded_noise(monkeypatch):
    """Replaces vd_vae.draw_noise by a queue of recorded tensors, consumed in decoder order."""
    from pytorch_generative_b200.models import vd_vae

    queue = []

    def draw(shape, device):
        e = queue.pop(0)
        assert tuple(e.shape) == tuple(shape), (e.shape, shape)
        return e.to(device)
    monkeypatch.setattr(vd_vae, "draw_noise", draw)
    return queue


def _gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / 2 ** 0.5))


def _dgelu64(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


# ----------------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------------
def test_gelu_cast_within_the_fit_error_and_into_a_column_range():
    """pg_gelu_cast uses pg_gelu_both: GELU within 3.2e-5 + 2^-12 |x| and GELU' within 1.2e-4 + 2^-11 of erf-GELU
    (pg_common.cuh), then one bf16 rounding (at most 2^-8 of the value).  Written into the second half of a wider operand, the
    first half is untouched and the pad columns are +0.0."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(0)
    x = (torch.randn(777, 13, generator=g) * 3).to(dev())
    a = torch.full((777, 32), 7.0, dtype=BF16, device=dev())
    d = torch.full((777, 32), 7.0, dtype=BF16, device=dev())
    L.gelu_cast(x, a[:, 13:], d[:, 13:])
    torch.cuda.synchronize()
    x64 = x.double()
    ga, da = a[:, 13:26].double(), d[:, 13:26].double()
    assert bool(((ga - _gelu64(x64)).abs() <= 2 ** -8 * _gelu64(x64).abs() + 3.3e-5 + 2 ** -12 * x64.abs()).all())
    assert bool(((da - _dgelu64(x64)).abs() <= 2 ** -8 * _dgelu64(x64).abs() + 1.3e-4 + 2 ** -11).all())
    assert bool((a[:, :13] == 7).all()) and bool((d[:, :13] == 7).all())
    for t in (a, d):
        pad = t[:, 26:].float()
        assert bool((pad == 0).all()) and not bool(torch.signbit(pad).any())


def _latent64(prior, post, x, eps, L_):
    C = x.shape[1]
    n = eps.shape[0]
    hw = eps[0, 0].numel()
    pm, pt, ph = prior[:, :L_], prior[:, L_:2 * L_], prior[:, 2 * L_:2 * L_ + C]
    e = eps.reshape(n, L_, hw).permute(0, 2, 1).reshape(n * hw, L_)
    if post is None:
        return pm + pt.exp() * e, x + ph, None
    qm, qs = post[:, :L_], post[:, L_:2 * L_]
    kl = R.gaussian_kl_div(qm, qs, pm, pt).reshape(n, hw * L_).sum(1)
    return qm + qs.exp() * e, x + ph, kl


@pytest.mark.parametrize("n,L_,side", [(1, 1, 1), (3, 3, 2), (128, 16, 1), (3, 16, 32), (128, 3, 2), (1, 16, 32)])
@pytest.mark.parametrize("sampling", [False, True])
def test_latent_kernels_against_float64(n, L_, side, sampling):
    """Forward: z within one bf16 rounding of the float64 value (plus the fp32 rounding of its terms), s = x + p_h
    within one fp32 rounding, kl within 1e-5 relative of its float64 sum (fp32 terms, at most 16K per image, summed in
    a fixed order) added to an existing kl.  Backward: against the float64 formulas within one bf16 rounding plus the
    fp32 error of exp and the quotients (2^-20 relative of the largest term); the bf16(dsum) columns bit for bit and
    the pad columns +0.0."""
    from pytorch_generative_b200 import _lib as L

    C = 12
    P = n * side * side
    g = torch.Generator().manual_seed(n * 100 + L_ * 10 + side)
    prior = (torch.randn(P, 2 * L_ + C + 3, generator=g) * 0.7).to(dev())
    post = None if sampling else (torch.randn(P, 2 * L_ + 1, generator=g) * 0.7).to(dev())
    x = torch.randn(P, C, generator=g).to(dev())
    eps = torch.randn(n, L_, side, side, generator=g).to(dev())
    kl_in = torch.randn(n, generator=g).to(dev())
    lp = -(-L_ // 8) * 8
    z = torch.full((P, lp), 5.0, dtype=BF16, device=dev())
    s = torch.empty(P, C, device=dev())
    kl = None if sampling else torch.empty(n, device=dev())
    L.vd_latent_fwd(prior, post, x, eps, z, s, kl_in, kl)
    z64, s64, kl64 = _latent64(prior.double(), None if post is None else post.double(), x.double(), eps.double(), L_)
    assert bool(((z[:, :L_].double() - z64).abs() <= 2 ** -8 * z64.abs() + 1e-6).all())
    assert bool((z[:, L_:].float() == 0).all()) and not bool(torch.signbit(z[:, L_:].float()).any())
    assert bool(((s.double() - s64).abs() <= 2 ** -23 * s64.abs()).all())
    if not sampling:
        want = kl_in.double() + kl64
        scale = R.gaussian_kl_div(post[:, :L_].double(), post[:, L_:2 * L_].double(), prior[:, :L_].double(),
                                  prior[:, L_:2 * L_].double()).abs().reshape(n, -1).sum(1)
        assert bool(((kl.double() - want).abs() <= 1e-5 * (scale + kl_in.double().abs()) + 1e-6).all())

    dz = torch.randn(P, lp, generator=g).to(dev(), BF16)
    g_kl = None if sampling else torch.randn(n, generator=g).to(dev())
    dsum = torch.randn(P, C, generator=g).to(dev())
    dprior = torch.full((P, -(-(2 * L_ + C) // 8) * 8), 5.0, dtype=BF16, device=dev())
    dpost = None if sampling else torch.full((P, -(-2 * L_ // 8) * 8), 5.0, dtype=BF16, device=dev())
    L.vd_latent_bwd(prior, post, eps, dz, g_kl, dsum, dprior, dpost)
    torch.cuda.synchronize()
    # float64 gradients by autograd through the same formulas
    pr = prior.double().requires_grad_()
    po = None if sampling else post.double().requires_grad_()
    z64, _, kl64 = _latent64(pr, po, x.double(), eps.double(), L_)
    obj = (z64 * dz[:, :L_].double()).sum() + (0 if sampling else (kl64 * g_kl.double()).sum())
    obj.backward()
    hw = side * side
    for got, ref, width in ((dprior, pr.grad, 2 * L_), (dpost, None if sampling else po.grad, 2 * L_)):
        if got is None:
            continue
        ref = ref[:, :width]
        # each entry is a sum of at most two products: bound by one bf16 rounding of the sum of their magnitudes
        mag = ref.abs() + (dz[:, :L_].double().abs().repeat(1, 2) * (1 + eps.double().reshape(n, L_, hw).permute(
            0, 2, 1).reshape(P, L_).abs().repeat(1, 2) * 3)) * 1e-6
        assert bool(((got[:, :width].double() - ref).abs() <= 2 ** -8 * ref.abs() + 1e-5 * (1 + mag)).all())
    assert torch.equal(dprior[:, 2 * L_:2 * L_ + C], dsum.to(BF16))
    for t, w in ((dprior, 2 * L_ + C), (dpost, 2 * L_)):
        if t is not None:
            pad = t[:, w:].float()
            assert bool((pad == 0).all()) and not bool(torch.signbit(pad).any())


@pytest.mark.parametrize("side", [1, 2, 3, 5, 8, 16, 32])
@pytest.mark.parametrize("C", [1, 12, 64, 100])
def test_pooling_against_float64(side, C):
    """Forward within one fp32 rounding of each sum step of the float64 mean (3 adds, exact quarter); odd sides are
    floored as nn.AvgPool2d does.  Backward: dy / 4 exactly under each window, +0.0 where no window covers."""
    from pytorch_generative_b200 import _lib as L

    n = 3
    g = torch.Generator().manual_seed(side * 1000 + C)
    x = torch.randn(n, C, side, side, generator=g, dtype=F64)
    x_pm = torch.empty(n * side * side, C, device=dev()).copy_(x.permute(0, 2, 3, 1).reshape(-1, C))
    ho = side // 2
    if ho == 0:
        return  # a 1-pixel side has no 2x2 window: pooling refuses it (h, w >= 2)
    y = torch.empty(n * ho * ho, C, device=dev())
    L.avg_pool2_fwd(x_pm, n, side, side, y)
    want = F.avg_pool2d(x_pm.double().cpu().reshape(n, side, side, C).permute(0, 3, 1, 2), 2, 2)
    want = want.permute(0, 2, 3, 1).reshape(-1, C)
    bound = 3 * 2 ** -24 * F.avg_pool2d(x_pm.double().cpu().reshape(n, side, side, C).permute(0, 3, 1, 2).abs(), 2, 2)
    assert bool(((y.double().cpu() - want).abs() <= bound.permute(0, 2, 3, 1).reshape(-1, C) + 1e-30).all())
    dy = torch.randn(n * ho * ho, C, generator=g).to(dev())
    dx = torch.full((n * side * side, C), 9.0, device=dev())
    L.avg_pool2_bwd(dy, n, side, side, dx)
    d4 = dx.cpu().reshape(n, side, side, C)
    up = (dy.cpu() / 4).reshape(n, ho, 1, ho, 1, C).expand(n, ho, 2, ho, 2, C).reshape(n, 2 * ho, 2 * ho, C)
    assert torch.equal(d4[:, :2 * ho, :2 * ho], up)
    rest = torch.cat([d4[:, 2 * ho:].reshape(-1), d4[:, :, 2 * ho:].reshape(-1)])
    assert bool((rest == 0).all()) and not bool(torch.signbit(rest).any())


@pytest.mark.parametrize("s", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("C", [1, 12, 64, 100])
@pytest.mark.parametrize("f", [1, 2])
@pytest.mark.parametrize("with_x", [True, False])
def test_bias_unpool_against_float64(s, C, f, with_x):
    """Forward: one fp32 addition, exactly the float64 sum rounded once.  Backward: dx = the sum of the f x f children
    and dbias = its sum over the images, within one fp32 rounding per addition of the float64 sums."""
    from pytorch_generative_b200 import _lib as L

    n = 5
    g = torch.Generator().manual_seed(s * 7 + C * 3 + f)
    bias = torch.randn(1, C, s, s, generator=g).to(dev())
    x = torch.randn(n * s * s, C, generator=g).to(dev()) if with_x else None
    S = s * f
    y = torch.empty(n * S * S, C, device=dev())
    L.bias_unpool_fwd(x, bias, n, f, y)
    b_pm = bias[0].permute(1, 2, 0).reshape(1, s, s, C)
    base = b_pm.expand(n, s, s, C) + (x.reshape(n, s, s, C) if with_x else 0)
    want = base.repeat_interleave(f, 1).repeat_interleave(f, 2).reshape(-1, C)
    assert torch.equal(y, want)
    dy = torch.randn(n * S * S, C, generator=g).to(dev())
    dx = torch.empty(n * s * s, C, device=dev()) if with_x else None
    dbias = torch.full((1, C, s, s), 3.0, device=dev())
    L.bias_unpool_bwd(dy, n, f, dx, dbias)
    d6 = dy.double().reshape(n, s, f, s, f, C)
    dx64 = d6.sum((2, 4))
    mag = dy.double().abs().reshape(n, s, f, s, f, C).sum((2, 4))
    if with_x:
        assert bool(((dx.double().reshape(n, s, s, C) - dx64).abs() <= f * f * 2 ** -24 * mag).all())
    db64 = dx64.sum(0).permute(2, 0, 1)[None]
    assert bool(((dbias.double() - db64).abs() <= (f * f + n) * 2 ** -24 * mag.sum(0).permute(2, 0, 1)[None]).all())


# ----------------------------------------------------------------------------------------------------------------------
# pm.conv with a GELU input
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,C,side,mode", [(1, 32, 8, "pointwise"), (3, 64, 16, "tap_loop"), (3, 32, 8, "gather"),
                                           (3, 32, 1, "gather"), (3, 32, 2, "gather"), (3, 12, 4, "gather")])
def test_conv_with_gelu_input_against_float64(k, C, side, mode):
    """y = conv(GELU(x)) + b + res and the PRE_GRAD GELU emit; dx = GELU'(x) (dy W), dw, db.  The float64 reference
    takes the device's bf16 operand a = bf16(GELU(x)) and stored derivative d, so the only device error left is the
    bf16 rounding of dy (2^-9) and fp32 accumulation: each output within 2^-8 of the sum of its terms' magnitudes."""
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.nn import pm

    n = 2
    g = torch.Generator().manual_seed(k * 100 + C + side)
    conv = torch.nn.Conv2d(C, C, k, padding=(k - 1) // 2).to(dev())
    geom = pm.Geom(n, side, side)
    x = torch.randn(n * side * side, C, generator=g).to(dev()).requires_grad_()
    res = torch.randn(n * side * side, C, generator=g).to(dev())
    xa = pm.gelu_operand(x)
    y, _ = pm.conv(x, conv.weight, conv.bias, geom, conv.padding, in_act=L.ACT_GELU, xa=xa, res=res, out_f32=True)
    assert y.shape == (n * side * side, C)
    from pytorch_generative_b200.nn.pm import GATHER, POINTWISE, TAP_LOOP  # noqa: F401
    dy = torch.randn(y.shape, generator=g).to(dev())
    y.backward(dy)
    a = xa.a[:, :C].double().reshape(n, side, side, C).permute(0, 3, 1, 2).requires_grad_()
    w64, b64 = conv.weight.detach().to(BF16).double().requires_grad_(), conv.bias.detach().double().requires_grad_()
    y64 = F.conv2d(a, w64, b64, padding=conv.padding).permute(0, 2, 3, 1).reshape(-1, C) + res.double()
    mag = F.conv2d(a.detach().abs(), w64.detach().abs(), b64.detach().abs(), padding=conv.padding).permute(
        0, 2, 3, 1).reshape(-1, C) + res.double().abs()
    assert bool(((y.double() - y64).abs() <= 2 ** -8 * mag + 1e-6).all())
    dyb = dy.to(BF16).double()
    y64.backward(dyb)
    dx64 = a.grad.permute(0, 2, 3, 1).reshape(-1, C) * xa.d[:, :C].double()
    dmag = F.conv_transpose2d(dyb.abs().reshape(n, side, side, C).permute(0, 3, 1, 2), w64.detach().abs(),
                              padding=conv.padding).permute(0, 2, 3, 1).reshape(-1, C) * xa.d[:, :C].double().abs()
    assert bool(((x.grad.double() - dx64).abs() <= 2 ** -7 * dmag + 1e-5).all())
    wmag = F.conv2d(a.detach().abs().transpose(0, 1), dyb.abs().reshape(n, side, side, C).permute(3, 0, 1, 2),
                    padding=conv.padding).transpose(0, 1)
    assert bool(((conv.weight.grad.double() - w64.grad).abs() <= 2 ** -7 * wmag + 1e-5).all())
    assert bool(((conv.bias.grad.double() - b64.grad).abs() <= 2 ** -7 * dyb.abs().sum(0) + 1e-5).all())


def test_conv_gelu_emit_feeds_the_next_conv():
    """A PRE_GRAD GELU emit: the next conv reads (GELU(y), GELU'(y)) from the producer's epilogue; the gradient of the
    producer's input equals the one through an explicit pg_gelu_cast of the fp32 y."""
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.nn import pm

    g = torch.Generator().manual_seed(3)
    C, n, side = 32, 2, 8
    geom = pm.Geom(n, side, side)
    c1, c2 = torch.nn.Conv2d(C, C, 1).to(dev()), torch.nn.Conv2d(C, C, 3, padding=1).to(dev())
    x = torch.randn(n * side * side, C, generator=g).to(dev())
    _, h = pm.conv(x, c1.weight, c1.bias, geom, in_act=L.ACT_GELU, emit=L.ACT_GELU, emit_mode=pm.PRE_GRAD,
                   want_main=False)
    yf, _ = pm.conv(x, c1.weight, c1.bias, geom, in_act=L.ACT_GELU, out_f32=True)
    ref = pm.gelu_operand(yf)
    assert torch.equal(h.a, ref.a) and torch.equal(h.d, ref.d)
    out, _ = pm.conv(h.a, c2.weight, c2.bias, geom, c2.padding, in_act=L.ACT_GELU, xa=h, out_f32=True)
    assert out.shape == (n * side * side, C) and bool(torch.isfinite(out).all())


# ----------------------------------------------------------------------------------------------------------------------
# the model
# ----------------------------------------------------------------------------------------------------------------------
def _loaded(case):
    from pytorch_generative_b200.models import vd_vae

    kwargs = dict(case["kwargs"])
    if case["stacks"] is not None:
        kwargs["stack_configs"] = [vd_vae.StackConfig(e, d) for e, d in case["stacks"]]
    m = vd_vae.VeryDeepVAE(**kwargs)
    m.load_state_dict(case["state"], strict=False)
    return m.to(dev())


def _cfg(case):
    stacks = case["stacks"] or [(1, 1)] * 6
    return case["kwargs"].get("input_resolution", 32), stacks, case["kwargs"].get("latent_channels", 4)


def _err(a, b):
    return (a.detach().double().cpu() - b.detach().double().cpu()).abs().max().item() / max(
        1.0, b.detach().double().abs().max().item())


TOL = 1e-2
# Each gradient is held to 5% of its own largest entry.  The float64 restatement does not take the device's bf16
# operands: every one of the up to ~30 convolutions on a gradient's path rounds its operands to bf16 (2^-9 relative),
# and the per-tensor maxima on the fixtures stay well below the bound (see the measured worst case in DESIGN).
GRAD_TOL = 5e-2


@pytest.mark.parametrize("name", ["default_32", "rgb_16"])
def test_the_reference_outputs_and_gradients(fixture, recorded_noise, name):
    from pytorch_generative_b200 import losses

    case = fixture[name]
    m = _loaded(case)
    x = case["x"].to(dev())
    recorded_noise.extend(case["eps"])
    logits, kl = m(x)
    assert not recorded_noise
    assert _err(logits, case["logits"]) <= TOL and _err(kl, case["kl"]) <= TOL
    loss = losses.vae_elbo(x, None, (logits, kl))
    for k, v in case["losses"].items():
        assert abs(loss[k].item() - v.item()) <= TOL * max(1.0, abs(v.item())), k
    loss["loss"].backward()
    g64, _, _, _ = R.grads({k: v for k, v in case["state"].items()}, case["x"], _cfg(case), case["eps"])
    worst = 0.0
    for k, p in m.named_parameters():
        ref = g64[k]
        e = (p.grad.double().cpu() - ref).abs().max().item() / max(1e-12, ref.abs().max().item())
        worst = max(worst, e)
        assert e <= GRAD_TOL, (k, e)
    print(f"{name}: worst per-tensor gradient error {worst:.4f}")


def test_recipe_widths_at_batch_4_against_the_fp32_restatement(recorded_noise):
    from pytorch_generative_b200 import losses
    from pytorch_generative_b200.models import VeryDeepVAE
    from pytorch_generative_b200.models.vd_vae import StackConfig

    stacks = [(3, 5), (3, 5), (2, 4), (2, 3), (2, 2), (1, 1)]
    torch.manual_seed(5)
    m = VeryDeepVAE(1, 1, 32, [StackConfig(*s) for s in stacks], latent_channels=16, hidden_channels=64,
                    bottleneck_channels=32).to(dev())
    g = torch.Generator().manual_seed(6)
    x = torch.bernoulli(torch.full((4, 1, 32, 32), 0.5), generator=g)
    eps = []
    for i, (_, nd) in enumerate(reversed(stacks)):
        side = 2 ** i
        eps += [torch.randn(4, 16, side, side, generator=g) for _ in range(nd)]
    recorded_noise.extend(eps)
    logits, kl = m(x.to(dev()))
    state = {k: v.cpu() for k, v in m.state_dict().items()}
    ref_logits, ref_kl = R.forward(state, x, (32, stacks, 16), eps)
    assert _err(logits, ref_logits) <= TOL and _err(kl, ref_kl) <= TOL
    losses.vae_elbo(x.to(dev()), None, (logits, kl))["loss"].backward()
    assert all(bool(torch.isfinite(p.grad).all()) for p in m.parameters())


def test_repeat_runs_are_bit_identical(fixture, recorded_noise):
    from pytorch_generative_b200 import losses

    case = fixture["rgb_16"]
    outs = []
    for _ in range(2):
        m = _loaded(case)
        recorded_noise.extend(case["eps"])
        x = case["x"].to(dev())
        logits, kl = m(x)
        losses.vae_elbo(x, None, (logits, kl))["loss"].backward()
        outs.append([logits, kl] + [p.grad for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_fused_adam_three_steps(fixture, recorded_noise):
    """Three FusedAdam steps against torch.optim.Adam on the fp32 restatement from the same state and noise: the
    losses agree within TOL at every step."""
    from pytorch_generative_b200 import losses, optim

    case = fixture["rgb_16"]
    m = _loaded(case)
    opt = optim.FusedAdam(m.parameters(), lr=5e-4)
    st = {k: v.clone().requires_grad_(True) for k, v in case["state"].items() if k in dict(m.named_parameters())}
    ref_opt = torch.optim.Adam(list(st.values()), lr=5e-4)
    x = case["x"].to(dev())
    for _ in range(3):
        recorded_noise.extend(case["eps"])
        opt.zero_grad()
        loss = losses.vae_elbo(x, None, m(x))["loss"]
        loss.backward()
        opt.clip_and_step(1e50)
        ref_opt.zero_grad()
        logits, kl = R.forward(st, case["x"], _cfg(case), case["eps"])
        ref_loss = R.elbo_loss(logits, kl, case["x"])
        ref_loss.backward()
        ref_opt.step()
        assert abs(loss.item() - ref_loss.item()) <= TOL * abs(ref_loss.item())


class _Preds(tuple):
    def detach(self):
        return _Preds(t.detach() for t in self)


class _TupleModel(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x):
        return _Preds(self.model(x))


def _tuple_loss(preds, x):
    from pytorch_generative_b200 import losses

    return losses.vae_elbo(x, None, preds)["loss"]


def test_graphed_train_step_equals_the_eager_step(fixture, monkeypatch):
    """The forward and backward never synchronise with the host, so the step captures as a CUDA graph; with the noise
    static tensors, two replays equal two eager steps bit for bit."""
    from pytorch_generative_b200 import trainstep
    from pytorch_generative_b200.models import vd_vae

    case = fixture["rgb_16"]
    eps = [e.to(dev()) for e in case["eps"]]
    counter = [0]

    def draw(shape, device):
        e = eps[counter[0] % len(eps)]
        counter[0] += 1
        return e
    monkeypatch.setattr(vd_vae, "draw_noise", draw)
    init = _loaded(case)
    state = {k: v.clone() for k, v in init.state_dict().items()}
    g = torch.Generator().manual_seed(8)
    xs = [torch.bernoulli(torch.full((2, 3, 16, 16), 0.5), generator=g).to(dev()) for _ in range(2)]
    graphed = _TupleModel(copy.deepcopy(init))
    step = trainstep.GraphedTrainStep(graphed, graphed.parameters(), _tuple_loss, xs[0], lr=1e-3, lr_gamma=1.0)
    step.reset({f"model.{k}": v for k, v in state.items()}, lr=1e-3)
    eager = _TupleModel(copy.deepcopy(init))
    eager.model.load_state_dict(state)
    params = list(eager.parameters())
    opt = torch.optim.Adam(params, lr=torch.tensor(1e-3, device=dev()), capturable=True)
    for x in xs:
        counter[0] = 0
        loss_g, norm_g = step(x)
        counter[0] = 0
        opt.zero_grad(set_to_none=True)
        loss = _tuple_loss(eager(x), x)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(params, 1e50, foreach=True)
        opt.step()
        assert loss_g == loss.item() and norm_g == norm.item()
    for (k, a), b in zip(graphed.named_parameters(), params):
        assert torch.equal(a.detach(), b.detach()), k


def test_sample_is_the_decoder_of_recorded_prior_noise_and_captures(fixture, recorded_noise):
    case = fixture["rgb_16"]
    m = _loaded(case)
    m._sample_fn = lambda t: t * 2
    n = case["x"].shape[0]
    recorded_noise.extend(case["sample_eps"])
    got = m.sample(n)
    assert not recorded_noise
    assert _err(got / 2, case["sample_logits"]) <= TOL
    # capturable: the whole of _sample replays as a CUDA graph with no host synchronisation
    static = [e.to(dev()) for e in case["sample_eps"]]
    recorded_noise.extend(static * 4)
    with torch.no_grad():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            m._sample(n)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m._sample(n)
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, got / 2)


def test_recipe_trains_one_epoch_and_checkpoints(tmp_path):
    from pytorch_generative_b200 import recipes

    g = torch.Generator().manual_seed(50)
    loader = [(torch.bernoulli(torch.full((8, 1, 32, 32), 0.5), generator=g).to(dev()), None) for _ in range(2)]
    trainer = recipes.reproduce_vd_vae(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["optimizer"]["param_groups"][0]["lr"] == 5e-4
    assert sorted(ckpt["model"]) == sorted(trainer.model.state_dict())
    assert bool(torch.isfinite(trainer.model.sample(4)).all())


def test_deepcopy_and_pickle_after_sample(fixture):
    m = _loaded(fixture["rgb_16"])
    m(fixture["rgb_16"]["x"].to(dev()))
    m.sample(2)
    for clone in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        for k, v in m.state_dict().items():
            assert torch.equal(clone.state_dict()[k], v)
