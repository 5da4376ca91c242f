"""NADE on the H100: probabilities and every gradient against float64 with per-element bounds (the recipe size and edge
shapes), the reference's own outputs (tests/golden/nade.pt) at the fp32 tolerance, bit-for-bit properties (repeat runs,
sub-batches, the autoregressive property, the checkpoints of `a`), forwards with entries to draw, sampling and the
recipe."""

import os

import pytest
import torch

import _nade_reference as R
from _checks import check

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nade.pt")
EPS = 2.0 ** -24  # fp32 unit roundoff
TOL = 1e-3        # the project's fp32 rule: relative to max(1, max|ref|)
F64 = torch.float64


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _model(kwargs, state, uniforms=None):
    from pytorch_generative_b200 import models

    m = models.NADE(**kwargs)
    m.load_state_dict(state)
    m = m.to(dev())
    if uniforms is not None:
        m._uniforms = lambda n, device: uniforms.to(device)
    return m


def _state(D, H, seed):
    """Default-initialised NADE(D, H) with some spread on the biases (so that relu(a) has both signs at d = 0)."""
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = models.NADE(D, H)
    with torch.no_grad():
        m._in_b.normal_(0, 0.5)
        m._h_b.normal_(0, 0.5)
    return {k: v.clone() for k, v in m.state_dict().items()}


def _input(shape, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "binary":
        return torch.bernoulli(torch.full(shape, 0.5), generator=g)
    return 2 * torch.rand(shape, generator=g)  # real-valued, >= 0: nothing to draw


# --------------------------------------------------------------------------------------------------
# float64 yardstick
# --------------------------------------------------------------------------------------------------
def _f64_reference(state, x, g):
    """p and every gradient of sum(g * p) in float64, with a per-element bound for the fp32 kernels.  The hidden
    pre-activations are the reference's float32 ones (the kernels reproduce their bits, see the checkpoint test), so
    the bounds cover the H-long dot, the sigmoid and the gradient sums: every rounding a result passes through, over
    the sum of the absolute terms of its chain, plus the error carried in from p."""
    n, D = x.shape
    p32 = {k: state[k].to(dev()) for k in R.PARAMS}
    A = R.hidden_preactivations(p32, x).to(F64)  # [n, D, H]
    H = A.shape[2]
    Wh, hb, Win = p32["_h_W"].to(F64), p32["_h_b"].to(F64), p32["_in_W"].to(F64)
    x64, g64 = x.to(F64), g.to(F64)
    relu = A.clamp_min(0)
    Z = torch.einsum("ndh,dh->nd", relu, Wh) + hb
    P = torch.sigmoid(Z)
    e_p = 0.25 * (H + 2) * EPS * (torch.einsum("ndh,dh->nd", relu, Wh.abs()) + hb.abs()) + 8 * EPS * P
    GZ = g64 * (1 - P) * P
    e_gz = g64.abs() * (1 - 2 * P).abs() * e_p + 4 * EPS * GZ.abs()
    out = {"p": (P, e_p)}
    out["_h_b"] = (GZ.sum(0), e_gz.sum(0) + n * EPS * GZ.abs().sum(0))
    out["_h_W"] = (torch.einsum("nd,ndh->dh", GZ, relu),
                   torch.einsum("nd,ndh->dh", e_gz, relu) + n * EPS * torch.einsum("nd,ndh->dh", GZ.abs(), relu))
    del relu
    mask = (A > 0).to(F64)
    del A
    DA = GZ[:, :, None] * Wh[None] * mask
    e_da = (e_gz[:, :, None] * Wh.abs()[None] + EPS * DA.abs()) * mask
    del mask

    def after(t):  # sum over d > i along dim 1
        inc = t.flip(1).cumsum(1).flip(1)
        return inc - t, inc[:, 0]

    S, S_all = after(DA)
    S_abs, S_abs_all = after(DA.abs())
    del DA
    E_s, E_s_all = after(e_da)
    del e_da
    E_s += D * EPS * S_abs
    E_s_all += D * EPS * S_abs_all
    out["_in_b"] = (S_all.sum(0), E_s_all.sum(0) + n * EPS * S_abs_all.sum(0))
    out["_in_W"] = (torch.einsum("ni,nih->hi", x64, S),
                    torch.einsum("ni,nih->hi", x64.abs(), E_s) + n * EPS * torch.einsum("ni,nih->hi", x64.abs(), S_abs))
    out["x"] = (torch.einsum("hi,nih->ni", Win, S),
                torch.einsum("hi,nih->ni", Win.abs(), E_s) + H * EPS * torch.einsum("hi,nih->ni", Win.abs(), S_abs))
    return out


CASES = [  # (n, D, H, image shape or None, input kind)
    (512, 784, 500, (1, 28, 28), "binary"),   # the recipe
    (37, 1, 10, None, "real"),
    (70, 37, 500, None, "binary"),            # n not a multiple of the image tile
    (33, 784, 1, (1, 28, 28), "binary"),
    (9, 64, 10, (1, 8, 8), "real"),
    (40, 64, 1000, None, "real"),
    (600, 37, 33, None, "binary"),            # 16 tiles of 38 images, the last one short
    (8, 64, 4096, (1, 8, 8), "binary"),
    (3, 40, 20000, None, "real"),             # wider than the registers hold: `a` in the scratch
]


@pytest.mark.parametrize("n,D,H,image,kind", CASES)
def test_forward_and_backward_against_float64(n, D, H, image, kind):
    state = _state(D, H, seed=D + H)
    x = _input((n, D), kind, seed=n).to(dev())
    g = torch.randn(n, D, generator=torch.Generator().manual_seed(7)).to(dev())
    m = _model(dict(input_dim=D, hidden_dim=H), state)
    xin = (x.view(n, *image) if image else x).clone().requires_grad_(True)
    p = m(xin)
    assert p.shape == xin.shape
    p.backward(g.view(p.shape))
    ref = _f64_reference(state, x, g)
    got = {"p": p.view(n, D), "x": xin.grad.view(n, D), **{k: prm.grad for k, prm in m.named_parameters()}}
    for name, (r, bound) in ref.items():
        check(f"{name} (n {n}, D {D}, H {H})", got[name].to(F64), r, 2 * bound)


@pytest.mark.parametrize("H", [77, 1000, 4096, 20000])  # one warp, 2 and 8 warps per image, `a` in the scratch
def test_checkpoints_carry_the_reference_bits(H):
    """The hidden pre-activations the forward keeps every NADE_CHUNK dimensions equal the reference's float32 ones, with
    entries drawn along the way; every draw compares its uniform with the probability the scan wrote."""
    from pytorch_generative_b200 import _lib as L

    n, D = 12, 100
    state = _state(D, H, seed=3)
    p32 = {k: state[k].to(dev()) for k in R.PARAMS}
    x = _input((n, D), "real", seed=4).to(dev())
    x[:, ::7] = -1.0  # drawn entries feed `a` too
    u = torch.rand(n, D, generator=torch.Generator().manual_seed(5)).to(dev())
    p = torch.empty(n, D, device=dev())
    xt = torch.empty_like(p)
    ckpt = torch.empty(n, -(-D // L.NADE_CHUNK), H, device=dev())
    L.nade_fwd(x, u, p32["_in_W"], p32["_in_b"], p32["_h_W"], p32["_h_b"], p, xt, ckpt)
    A = R.hidden_preactivations(p32, xt)
    assert torch.equal(ckpt, A[:, ::L.NADE_CHUNK])
    assert torch.equal(xt[x >= 0], x[x >= 0])
    drawn = x < 0
    assert torch.equal(xt[drawn], (u < p).float()[drawn])


def test_grad_free_calls_keep_no_checkpoints(monkeypatch):
    """sample() and forwards under no_grad write no checkpoints (a forward with gradients does)."""
    from pytorch_generative_b200 import _lib as L

    kept = []
    real = L.nade_fwd
    monkeypatch.setattr(L, "nade_fwd", lambda *a, **k: (kept.append(a[8] is not None), real(*a, **k))[1])
    m = _model(dict(input_dim=64, hidden_dim=32), _state(64, 32, seed=1))
    x = _input((4, 64), "binary", seed=2).to(dev())
    m.sample(conditioned_on=-torch.ones_like(x))
    with torch.no_grad():
        m(x)
    m(x)
    assert kept == [False, False, True]


def test_an_empty_batch():
    """n = 0 through the kernels: empty p and x~, zero gradients (the reference's `_forward` returns empty tensors)."""
    m = _model(dict(input_dim=64, hidden_dim=32), _state(64, 32, seed=1))
    x = torch.zeros(0, 64, device=dev(), requires_grad=True)
    p, xt = m._forward(x)
    assert p.shape == xt.shape == (0, 64)
    p.sum().backward()
    assert x.grad.shape == (0, 64)
    assert all(bool((prm.grad == 0).all()) for prm in m.parameters())


# --------------------------------------------------------------------------------------------------
# The reference's own outputs
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["image_192_10", "image_64_32", "vector_37_1"])
@pytest.mark.parametrize("kind", ["binary", "negative"])
def test_fixture_forward_and_gradients(fixture, name, kind):
    from pytorch_generative_b200 import losses

    fx = fixture[name]
    f = fx[kind]
    m = _model(fx["kwargs"], fx["state"], f["uniforms"])
    x = f["x"].to(dev()).requires_grad_(True)
    p = m(x)
    loss = losses.bce_with_logits_sum_mean(p, x.detach())
    loss.backward()
    report = {"p": _err(p, f["p"]), "loss": _err(loss, f["loss"]), "x grad": _err(x.grad, f["x_grad"])}
    for k, prm in m.named_parameters():
        report[k] = _err(prm.grad, f["grads"][k])
    assert max(report.values()) <= TOL, report
    drawn = f["x"] < 0
    assert bool((x.grad.cpu()[drawn] == 0).all())


# --------------------------------------------------------------------------------------------------
# Bit-for-bit properties
# --------------------------------------------------------------------------------------------------
def _run(m, x):
    m.zero_grad()
    p = m(x)
    p.backward(torch.ones_like(p))
    return p.detach().clone(), {k: prm.grad.clone() for k, prm in m.named_parameters()}


def test_repeat_runs_sub_batches_and_the_autoregressive_property():
    n, D, H = 96, 784, 500
    state = _state(D, H, seed=11)
    m = _model(dict(input_dim=D, hidden_dim=H), state)
    x = _input((n, D), "binary", seed=12).to(dev())
    p1, g1 = _run(m, x)
    p2, g2 = _run(m, x)
    assert torch.equal(p1, p2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    with torch.no_grad():
        assert torch.equal(m(x[17:40]), p1[17:40])
        assert torch.equal(m(x[5:6]), p1[5:6])
        for d in (0, 1, 15, 16, 17, 400, 783):
            changed = x.clone()
            changed[:, d:] = 1 - changed[:, d:]
            assert torch.equal(m(changed)[:, : d + 1], p1[:, : d + 1]), d


def test_a_draw_at_the_last_dimension_leaves_every_probability_alone():
    """An image whose only negative entry is its last dimension: the same probabilities as without it (the draw comes
    after the last probability), and x~ keeps every given entry."""
    D, H = 784, 500
    m = _model(dict(input_dim=D, hidden_dim=H), _state(D, H, seed=13))
    x = _input((6, D), "binary", seed=14).to(dev())
    with torch.no_grad():
        base = m(x)
        x_neg = x.clone()
        x_neg[2, -1] = -1.0
        assert torch.equal(m(x_neg), base)
        xt = m._forward(x_neg)[1]
    assert torch.equal(xt[:, :-1], x[:, :-1]) and xt[2, -1].item() in (0.0, 1.0)


# --------------------------------------------------------------------------------------------------
# Sampling
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["image_192_10", "image_64_32", "vector_37_1"])
def test_sampling_under_recorded_uniforms_matches_the_reference(fixture, name):
    """The reference's own samples, up to a knife-edge draw (|u - p| within the fp32 tolerance) and what follows it;
    given entries come back bit for bit."""
    fx = fixture[name]
    for kind in ("unconditional", "conditional"):
        s = fx[kind]
        m = _model(fx["kwargs"], fx["state_after"], s["uniforms"])
        ref = s["sample"]
        if s["conditioned_on"] is None:
            got = m.sample(ref.shape[0]).cpu()
            start = -torch.ones_like(ref)
        else:
            got = m.sample(conditioned_on=s["conditioned_on"].to(dev())).cpu()
            start = s["conditioned_on"]
            given = start >= 0
            assert torch.equal(got[given], start[given])
        assert got.shape == ref.shape
        n = ref.shape[0]
        diff = (got.view(n, -1) != ref.view(n, -1)).any(0)
        if diff.any():
            first = int(diff.nonzero()[0])
            state = {k: fx["state_after"][k] for k in R.PARAMS}
            probs = R.forward(state, ref.view(n, -1).clone(), s["uniforms"])[0][:, first]
            margin = (s["uniforms"][:, first] - probs).abs().min().item()
            assert margin < TOL, f"{kind}: samples diverge at dimension {first} without a knife-edge draw ({margin:.3e})"


@pytest.mark.parametrize("D", [64, 784])
def test_sample_launches_a_fixed_number_of_kernels(D):
    from pytorch_generative_b200 import _lib as L

    m = _model(dict(input_dim=D, hidden_dim=500), _state(D, 500, seed=D))
    canvas = -torch.ones(16, D, device=dev())
    m.sample(conditioned_on=canvas)
    before = L.launch_count()
    out = m.sample(conditioned_on=canvas)
    torch.cuda.synchronize()
    assert L.launch_count() - before == 2  # the transpose of _in_W and the scan
    assert bool(((out == 0) | (out == 1)).all())


def test_auto_reshape_behaviours():
    m = _model(dict(input_dim=192, hidden_dim=10), _state(192, 10, seed=2))
    x = _input((4, 3, 8, 8), "binary", seed=3).to(dev())
    assert m(x).shape == (4, 3, 8, 8) and int(m._c) == 3 and int(m._h) == 8 and int(m._w) == 8
    assert m.sample(n_samples=2).shape == (2, 3, 8, 8)
    cond = torch.where(x < 0.5, -torch.ones_like(x), x)
    out = m.sample(conditioned_on=cond)
    assert out.shape == (4, 3, 8, 8) and torch.equal(out[cond >= 0], cond[cond >= 0])


# --------------------------------------------------------------------------------------------------
# Training
# --------------------------------------------------------------------------------------------------
def test_fused_adam_trajectory_matches_the_restatement(fixture):
    from pytorch_generative_b200 import losses, optim

    fx = fixture["image_64_32"]
    m = _model(fx["kwargs"], fx["state"])
    ref = R.TrainState(fx["state"])
    opt = optim.FusedAdam(m.parameters())
    for s in range(3):
        x = _input((16, 1, 8, 8), "binary", seed=20 + s)
        ref_loss, ref_norm = ref.step(x, torch.zeros(16, 64))
        xd = x.to(dev())
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(m(xd), xd)
        loss.backward()
        norm = opt.clip_and_step(1e50).item()
        assert abs(loss.item() - ref_loss) <= TOL * max(1.0, abs(ref_loss)), (s, loss.item(), ref_loss)
        assert abs(norm - ref_norm) <= TOL * ref_norm, (s, norm, ref_norm)
    for k, prm in m.named_parameters():
        assert _err(prm, ref.p[k]) <= TOL, k


def test_reproduce_nade_trains_checkpoints_and_reloads(tmp_path):
    from pytorch_generative_b200 import models, recipes

    loader = [(_input((64, 1, 28, 28), "binary", seed=30 + i).to(dev()), None) for i in range(2)]
    trainer = recipes.reproduce_nade(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["optimizer"]["param_groups"][0]["lr"] == 1e-3 and "lr_scheduler" not in ckpt
    fresh = models.NADE(784, 500)
    fresh.load_state_dict(ckpt["model"])
    for k, v in trainer.model.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v.cpu()), k


def test_reproduce_nade_on_randn_images_has_a_finite_loss(tmp_path):
    """The reference's integration test feeds torch.randn images: every negative entry is drawn inside the forward."""
    from pytorch_generative_b200 import recipes

    g = torch.Generator().manual_seed(40)
    loader = [(torch.randn(8, 1, 28, 28, generator=g).to(dev()), None) for _ in range(2)]
    trainer = recipes.reproduce_nade(n_epochs=1, batch_size=8, log_dir=str(tmp_path), debug_loader=loader)
    for prm in trainer.model.parameters():
        assert bool(torch.isfinite(prm).all())
    with torch.no_grad():
        x = loader[0][0]
        p = trainer.model(x)
        from pytorch_generative_b200 import losses

        assert bool(torch.isfinite(losses.bce_with_logits_sum_mean(p, x)))
