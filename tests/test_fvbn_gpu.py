"""FVBN on the H100: logits and every gradient against float64 with per-element bounds (D in {1, 2, 37, 100, 784, 3072},
n in {1, 5, 300, 512}), the reference's own outputs (tests/golden/fvbn.pt) at the fp32 tolerance, bit-for-bit properties
(repeat runs, sub-batches, the autoregressive property), the sampler (teacher-forced logits against the forward on the
canvas at every step, graph replay, reference samples under recorded uniforms), launch counts, a FusedAdam trajectory
and the recipe."""

import copy
import os
import pickle

import pytest
import torch

import _fvbn_reference as R
from _checks import check

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fvbn.pt")
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


def _model(D, seed, sample_fn=None):
    """Default-initialised FVBN(D) under `seed`, biases spread by N(0, 0.5), on the GPU."""
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = models.FullyVisibleBeliefNetwork(D, sample_fn=sample_fn)
    with torch.no_grad():
        for row in m._net:
            row.bias.normal_(0, 0.5)
    return m.to(dev())


def _loaded(kwargs, state, sample_fn=None):
    from pytorch_generative_b200 import models

    m = models.FullyVisibleBeliefNetwork(**kwargs, sample_fn=sample_fn)
    m.load_state_dict(state)
    return m.to(dev())


def _input(shape, kind, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.bernoulli(torch.full(shape, 0.5), generator=g)
    if kind == "randn":
        x = torch.randn(shape, generator=g)
    elif kind == "negative":  # 0/1 with about 30% of the entries -1, as an unfinished sampling canvas holds them
        x = torch.where(torch.rand(shape, generator=g) < 0.3, -torch.ones(shape), x)
    return x


# --------------------------------------------------------------------------------------------------
# float64 yardstick
# --------------------------------------------------------------------------------------------------
def _f64_reference(state, x, g):
    """Logits and every gradient of sum(g * logits) in float64, each with a per-element bound for the fp32 kernels:
    gamma_k * (sum of the absolute terms) for a k-long chain of roundings (k = the sum's length plus the bias add, or plus
    the slice partials added by pg_sum_partials)."""
    n, D = x.shape
    p = {k: v.to(dev(), F64) for k, v in state.items() if k.startswith("_net.")}
    W, w0, b = R.dense(p, D)  # W [D, D] strictly lower triangular
    x64, g64 = x.to(dev(), F64), g.to(dev(), F64)
    gamma = lambda k: k * EPS / (1 - k * EPS)
    rows = torch.arange(D, device=dev(), dtype=F64)
    logits = x64 @ W.t() + b
    logits[:, 0] = b[0] + w0[0] * 0.0
    e_logits = gamma(rows + 2) * ((x64.abs() @ W.abs().t()) + b.abs())
    out = {"logits": (logits, e_logits)}
    dW = (g64.t() @ x64).tril(-1)
    e_dW = gamma(n + 34) * (g64.abs().t() @ x64.abs()).tril(-1)
    off, T = R.offsets(D)
    packed, e_packed = torch.zeros(T, dtype=F64, device=dev()), torch.zeros(T, dtype=F64, device=dev())
    for i in range(1, D):
        packed[off[i]: off[i] + i] = dW[i, :i]
        e_packed[off[i]: off[i] + i] = e_dW[i, :i]
    out["weights"] = (packed, e_packed)  # row 0's entry: sum_b g * 0 = 0 exactly
    out["biases"] = (g64.sum(0), gamma(n + 34) * g64.abs().sum(0))
    if D > 1:
        out["x"] = (g64 @ W, gamma(D + 1) * (g64.abs() @ W.abs()))
    return out


def _packed_grads(m):
    """The model's gradients as (packed weight gradient [T], bias gradient [D])."""
    ws = torch.cat([row.weight.grad.reshape(-1) for row in m._net])
    bs = torch.cat([row.bias.grad.reshape(-1) for row in m._net])
    return ws, bs


CASES = [  # (n, D, image shape or None, input kind)
    (1, 1, None, "randn"),
    (5, 1, (1, 1, 1), "binary"),
    (512, 2, None, "negative"),
    (5, 37, None, "randn"),
    (512, 37, None, "binary"),
    (300, 100, None, "negative"),          # three batch slices of 100 images, tiles cut at n and D
    (1, 784, (1, 28, 28), "binary"),
    (512, 784, (1, 28, 28), "binary"),     # the recipe
    (512, 784, None, "negative"),
    (5, 784, None, "randn"),
    (5, 3072, (3, 32, 32), "randn"),
    (512, 3072, (3, 32, 32), "binary"),
]


@pytest.mark.parametrize("n,D,image,kind", CASES)
def test_forward_and_backward_against_float64(n, D, image, kind):
    m = _model(D, seed=D + n)
    state = m.state_dict()
    x = _input((n, D), kind, seed=n).to(dev())
    g = torch.randn(n, D, generator=torch.Generator().manual_seed(7)).to(dev())
    xin = (x.view(n, *image) if image else x).clone().requires_grad_(True)
    logits = m(xin)
    assert logits.shape == xin.shape
    logits.backward(g.view(logits.shape))
    ref = _f64_reference(state, x, g)
    ws, bs = _packed_grads(m)
    got = {"logits": logits.view(n, D), "weights": ws, "biases": bs}
    if D > 1:
        got["x"] = xin.grad.view(n, D)
    else:
        assert xin.grad is None  # the input feeds no row, as in the reference
    for name, (r, bound) in ref.items():
        check(f"{name} (n {n}, D {D}, {kind})", got[name].to(F64), r, 2 * bound)


def test_row_zero_propagates_a_non_finite_weight():
    """Row 0's logit is b_0 + w_0 * 0 computed, as in the reference: an infinite w_0 makes it NaN (and only it)."""
    m = _model(8, seed=1)
    with torch.no_grad():
        m._net[0].weight.fill_(float("inf"))
        out = m(_input((3, 8), "binary", seed=2).to(dev()))
    assert bool(out[:, 0].isnan().all()) and bool(out[:, 1:].isfinite().all())


def test_an_empty_batch_through_the_kernels():
    """n = 0 does nothing: no logits, nothing added to the gradients.  (The model itself refuses an empty batch in
    `x.view(0, -1)`, as the reference does.)"""
    from pytorch_generative_b200 import _lib as L

    m = _model(37, seed=3)
    layout, table = m._table(m._params())
    x = torch.zeros(0, 37, device=dev())
    L.fvbn_fwd(table, x, torch.empty(0, 37, device=dev()))
    buf = torch.zeros(layout.total + 37, device=dev())
    L.fvbn_bwd(table, x, torch.zeros(0, 37, device=dev()), buf[: layout.total], buf[layout.total:],
               torch.empty(0, 37, device=dev()))
    torch.cuda.synchronize()
    assert bool((buf == 0).all())


def test_the_table_follows_the_parameters():
    """Parameters moved to fresh storage (the old storage kept alive, so no address can be reused): the key changes,
    the same table tensor is rewritten in place with the new addresses, and the logits are unchanged."""
    m = _model(100, seed=4)
    x = _input((9, 100), "binary", seed=5).to(dev())
    with torch.no_grad():
        before = m(x)
        table = m._fvbn_table.table([r.weight for r in m._net], [r.bias for r in m._net])
        old_key = m._fvbn_table._tables[dev()][0]
        old = [p.data for p in m.parameters()]
        for p in m.parameters():
            p.data = p.data.clone()
        after = m(x)
    new_key = m._fvbn_table._tables[dev()][0]
    assert new_key != old_key and new_key == tuple(p.data_ptr() for p in m._params()[0::2] + m._params()[1::2])
    assert m._fvbn_table._tables[dev()][1] is table and table.tolist() == list(new_key)
    assert torch.equal(before, after)
    assert all(t.data_ptr() not in new_key for t in old)


@pytest.mark.parametrize("convert", ["half", "bfloat16", "double"])
def test_parameters_of_another_dtype_are_refused(convert):
    """The kernels read fp32 rows: after .half() / .bfloat16() / .double() the rebuild of the table refuses the
    parameters before any launch."""
    from pytorch_generative_b200 import _lib as L

    m = _model(37, seed=6)
    x = _input((4, 37), "binary", seed=7).to(dev())
    m(x)  # a table for the fp32 parameters
    getattr(m, convert)()
    before = L.launch_count()
    with pytest.raises(RuntimeError, match="contiguous fp32"):
        m(x)
    with pytest.raises(RuntimeError, match="contiguous fp32"):
        m.sample(conditioned_on=-torch.ones(2, 1, 1, 37, device=dev()))
    assert L.launch_count() == before


def test_a_parameter_of_the_wrong_size_is_refused():
    m = _model(8, seed=8)
    with torch.no_grad():
        m._net[5].weight.data = torch.zeros(1, 4, device=dev())
    with pytest.raises(RuntimeError, match=r"_net\.5\.weight .* 4 elements \(expected 5"):
        m(_input((2, 8), "binary", seed=9).to(dev()))


def test_the_backward_adds_the_same_bits_into_separate_gradient_buffers():
    """pg_fvbn_bwd sums its partials once when db follows dw in memory and once per output otherwise: same bits."""
    from pytorch_generative_b200 import _lib as L

    n, D = 300, 100
    m = _model(D, seed=10)
    layout, table = m._table(m._params())
    x = _input((n, D), "negative", seed=11).to(dev())
    g = torch.randn(n, D, generator=torch.Generator().manual_seed(12)).to(dev())
    joint = torch.zeros(layout.total + D, device=dev())
    dx1, dx2 = torch.empty(n, D, device=dev()), torch.empty(n, D, device=dev())
    L.fvbn_bwd(table, x, g, joint[: layout.total], joint[layout.total:], dx1)
    dw, db = torch.zeros(layout.total, device=dev()), torch.zeros(D, device=dev())
    L.fvbn_bwd(table, x, g, dw, db, dx2)
    assert torch.equal(joint[: layout.total], dw) and torch.equal(joint[layout.total:], db) and torch.equal(dx1, dx2)


# --------------------------------------------------------------------------------------------------
# The reference's own outputs
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["image_1x8x8", "image_3x4x4", "image_1x1x1"])
@pytest.mark.parametrize("kind", ["binary", "negative"])
def test_fixture_forward_and_gradients(fixture, name, kind):
    from pytorch_generative_b200 import losses

    fx = fixture[name]
    f = fx[kind]
    m = _loaded(fx["kwargs"], fx["state"])
    x = f["x"].to(dev()).requires_grad_(True)
    logits = m(x)
    loss = losses.bce_with_logits_sum_mean(logits, x.detach())
    loss.backward()
    report = {"logits": _err(logits, f["logits"]), "loss": _err(loss, f["loss"])}
    if f["x_grad"] is None:
        assert x.grad is None
    else:
        report["x grad"] = _err(x.grad, f["x_grad"])
    for k, prm in m.named_parameters():
        report[k] = _err(prm.grad, f["grads"][k])
    assert max(report.values()) <= TOL, report


# --------------------------------------------------------------------------------------------------
# Bit-for-bit properties
# --------------------------------------------------------------------------------------------------
def _run(m, x):
    m.zero_grad()
    logits = m(x)
    logits.backward(torch.ones_like(logits))
    return logits.detach().clone(), {k: prm.grad.clone() for k, prm in m.named_parameters()}


def test_repeat_runs_sub_batches_and_the_autoregressive_property():
    n, D = 512, 784
    m = _model(D, seed=11)
    x = _input((n, D), "binary", seed=12).to(dev())
    l1, g1 = _run(m, x)
    l2, g2 = _run(m, x)
    assert torch.equal(l1, l2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    with torch.no_grad():
        assert torch.equal(m(x[17:40]), l1[17:40])
        assert torch.equal(m(x[5:6]), l1[5:6])
        for d in (0, 1, 31, 32, 33, 400, 783):
            changed = x.clone()
            changed[:, d:] = 1 - changed[:, d:]
            assert torch.equal(m(changed)[:, : d + 1], l1[:, : d + 1]), d


@pytest.mark.parametrize("D", [37, 784, 3072])
def test_forward_and_backward_launch_a_fixed_number_of_kernels(D):
    from pytorch_generative_b200 import _lib as L

    m = _model(D, seed=D)
    x = _input((8, D), "binary", seed=1).to(dev()).requires_grad_(True)
    m(x).sum().backward()  # warm-up: the scratch grows outside the count
    torch.cuda.synchronize()
    before = L.launch_count()
    m(x).sum().backward()
    torch.cuda.synchronize()
    assert L.launch_count() - before == 3  # the forward; the backward's tile kernel and its one sum


# --------------------------------------------------------------------------------------------------
# Sampling
# --------------------------------------------------------------------------------------------------
def _recorder(draw=lambda logits: torch.zeros_like(logits)):
    calls = []

    def fn(logits):
        calls.append(logits.detach().clone())
        return draw(logits)

    return calls, fn


@pytest.mark.parametrize("shape", [(16, 1, 28, 28), (5, 3, 4, 4)])
def test_teacher_forced_sampling_matches_the_forward(shape):
    """Every entry given: sample_fn sees h*w calls of [n, c] logits, bit-equal to the forward's at that pixel, and the
    canvas comes back unchanged; a second call replays the captured step with the same logits."""
    n, c, h, w = shape
    calls, fn = _recorder()
    m = _model(c * h * w, seed=21, sample_fn=fn)
    x = _input(shape, "binary", seed=22).to(dev())
    with torch.no_grad():
        full = m(x)
    runs = []
    for _ in range(2):
        calls.clear()
        out = m.sample(conditioned_on=x)
        assert torch.equal(out, x)
        assert len(calls) == h * w and all(cl.shape == (n, c) for cl in calls)
        for p, cl in enumerate(calls):
            assert torch.equal(cl, full[:, :, p // w, p % w]), p
        runs.append(torch.stack(calls))
    assert torch.equal(runs[0], runs[1])
    assert all(st["graph"] is not None for st in m._fvbn_sampler.values())


@pytest.mark.parametrize("shape", [(16, 1, 28, 28), (5, 3, 4, 4)])
def test_sampling_logits_come_from_the_live_canvas(shape):
    """Entries to draw (-1) mixed with given ones: each call's logits are bit-equal to the forward of the canvas as it
    stands at that step (for c > 1 the later channels of the pixel still -1), and given entries come back bit for bit."""
    n, c, h, w = shape
    calls, fn = _recorder(lambda logits: (logits > 0).float())
    m = _model(c * h * w, seed=23, sample_fn=fn)
    start = _input(shape, "negative", seed=24).to(dev())
    out = m.sample(conditioned_on=start)
    given = start >= 0
    assert torch.equal(out[given], start[given]) and bool(((out == 0) | (out == 1)).all())
    canvas = start.clone()
    with torch.no_grad():
        for p, cl in enumerate(calls):
            r, col = divmod(p, w)
            assert torch.equal(cl, m(canvas)[:, :, r, col]), p
            cur = canvas[:, :, r, col]
            canvas[:, :, r, col] = torch.where(cur < 0, (cl > 0).float(), cur)
    assert torch.equal(canvas, out)


@pytest.mark.parametrize("name", ["image_1x8x8", "image_3x4x4", "image_1x1x1"])
def test_sampling_under_recorded_uniforms_matches_the_reference(fixture, name):
    """The reference's own samples, up to a knife-edge draw (|u - sigmoid(logit)| within the fp32 logit bound) and what
    follows it; given entries come back bit for bit."""
    fx = fixture[name]
    D = fx["kwargs"]["n_dims"]
    for kind in ("unconditional", "conditional"):
        s = fx[kind]
        m = _loaded(fx["kwargs"], fx["state_after"], R.uniform_sample_fn(s["uniforms"]))
        ref = s["sample"]
        n, c, h, w = ref.shape
        if s["conditioned_on"] is None:
            got = m.sample(n).cpu()
            start = -torch.ones_like(ref)
        else:
            start = s["conditioned_on"]
            got = m.sample(conditioned_on=start.to(dev())).cpu()
            assert torch.equal(got[start >= 0], start[start >= 0])
        assert got.shape == ref.shape
        diff = (got != ref).any(1).any(0).view(-1)  # per pixel, raster order
        if diff.any():
            first = int(diff.nonzero()[0])
            canvas = start.clone().to(F64)
            done = torch.arange(h * w).view(h, w) < first
            canvas[:, :, done] = ref[:, :, done].to(F64)
            p = {k: v.to(F64) for k, v in fx["state_after"].items() if k.startswith("_net.")}
            logits = R.forward(p, canvas.view(n, D)).view(n, c, h, w)[:, :, first // w, first % w]
            margin = (s["uniforms"][first].to(F64) - torch.sigmoid(logits)).abs().min().item()
            assert margin < 1e-4, f"{kind}: samples diverge at pixel {first} without a knife-edge draw ({margin:.3e})"


def _threshold(logits):
    return (logits > 0).float()


def test_deepcopy_and_pickle_after_sample():
    m = _model(48, seed=31, sample_fn=_threshold)  # a module-level sample_fn: the model pickles
    m(_input((2, 3, 4, 4), "binary", seed=32).to(dev()))  # registers the image shape
    first = m.sample(3)
    twin = copy.deepcopy(m)
    assert "_fvbn_sampler" not in twin.__dict__ and "_fvbn_table" not in twin.__dict__
    assert torch.equal(twin.sample(3), first) and torch.equal(m.sample(3), first)
    clone = pickle.loads(pickle.dumps(m))
    assert "_fvbn_sampler" not in clone.__dict__
    assert torch.equal(clone.sample(3), first)


# --------------------------------------------------------------------------------------------------
# Training
# --------------------------------------------------------------------------------------------------
def test_fused_adam_trajectory_matches_the_restatement(fixture):
    from pytorch_generative_b200 import losses, optim

    fx = fixture["image_1x8x8"]
    m = _loaded(fx["kwargs"], fx["state"])
    ref = R.TrainState(fx["state"])
    opt = optim.FusedAdam(m.parameters())
    for s in range(3):
        x = _input((16, 1, 8, 8), "binary", seed=20 + s)
        ref_loss, ref_norm = ref.step(x)
        xd = x.to(dev())
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(m(xd), xd)
        loss.backward()
        norm = opt.clip_and_step(1e50).item()
        assert abs(loss.item() - ref_loss) <= TOL * max(1.0, abs(ref_loss)), (s, loss.item(), ref_loss)
        assert abs(norm - ref_norm) <= TOL * ref_norm, (s, norm, ref_norm)
    for k, prm in m.named_parameters():
        assert _err(prm, ref.p[k]) <= TOL, k


def test_reproduce_fvbn_trains_checkpoints_and_reloads(tmp_path):
    from pytorch_generative_b200 import models, recipes

    loader = [(_input((64, 1, 28, 28), "binary", seed=30 + i).to(dev()), None) for i in range(2)]
    trainer = recipes.reproduce_fvbn(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["optimizer"]["param_groups"][0]["lr"] == 1e-3 and "lr_scheduler" not in ckpt
    fresh = models.FullyVisibleBeliefNetwork(784)
    fresh.load_state_dict(ckpt["model"])
    for k, v in trainer.model.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v.cpu()), k
    for prm in trainer.model.parameters():
        assert bool(torch.isfinite(prm).all())
