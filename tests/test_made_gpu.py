"""MADE on the H100: the mask-and-cast kernel bit for bit, forward / loss / every gradient against the float32 restatement
(tests/_made_reference.py) and the reference's own outputs (tests/golden/made.pt), the autoregressive property, a FusedAdam
trajectory, the incremental sampler (teacher forcing, graph replay, pre-drawn uniforms) and the recipe."""

import os

import numpy as np
import pytest
import torch

import _made_reference as R

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "made.pt")
TOL = 1e-2  # bf16 operands, fp32 accumulation: relative to max(1, max|ref|)


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _model(kwargs, state, sample_fn=None):
    from pytorch_generative_b200 import models

    m = models.MADE(**kwargs, sample_fn=sample_fn)
    m.load_state_dict({k: v for k, v in state.items() if k not in ("_c", "_h", "_w")}, strict=False)
    return m.to(dev())


def _recipe_state(seed=0):
    """Default-initialised MADE(784, [8000]) weights (the recipe's model) with some spread on the biases."""
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = models.MADE(784, [8000])
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape) * 0.01)
    return {k: v.clone() for k, v in m.state_dict().items()}


def _binary(shape, seed):
    return torch.bernoulli(torch.full(shape, 0.5), generator=torch.Generator().manual_seed(seed))


# --------------------------------------------------------------------------------------------------
# pg_made_mask_cast
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,strict", [(37, 29, 0), (37, 29, 1), (64, 784, 0), (784, 64, 1)])
def test_mask_cast_is_bit_exact(rows, cols, strict):
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(rows * cols + strict)
    w = torch.randn(rows, cols, generator=g)
    c_in = torch.randint(0, 50, (cols,), generator=g, dtype=torch.int32)
    c_out = torch.randint(0, 50, (rows,), generator=g, dtype=torch.int32)
    mask = ((c_in[None, :] < c_out[:, None]) if strict else (c_in[None, :] <= c_out[:, None])).float()
    want_w = w * mask
    rp, cp = (rows + 7) // 8 * 8, (cols + 7) // 8 * 8
    want_q = torch.zeros(rp, cp, dtype=torch.bfloat16)
    want_q[:rows, :cols] = want_w.bfloat16()

    wd = w.to(dev())
    version = wd._version
    q = torch.full((rp, cp), 7.0, dtype=torch.bfloat16, device=dev())
    buf = torch.full((rows, cols), 5.0, device=dev())
    L.made_mask_cast(wd, c_in.to(dev()), c_out.to(dev()), strict, q, buf)
    torch.cuda.synchronize()
    assert torch.equal(wd.cpu(), want_w) and torch.equal(wd.cpu().signbit(), want_w.signbit())
    assert torch.equal(q.cpu(), want_q)
    assert torch.equal(buf.cpu(), mask)
    assert wd._version == version
    buf.fill_(5.0)
    q.fill_(7.0)
    L.made_mask_cast(wd, c_in.to(dev()), c_out.to(dev()), strict, q, None)  # no mask buffer: left alone
    assert torch.equal(wd.cpu(), want_w) and torch.equal(q.cpu(), want_q)
    assert bool((buf == 5.0).all())


# --------------------------------------------------------------------------------------------------
# Training path
# --------------------------------------------------------------------------------------------------
def _check_step(m, x, ref_logits, ref_loss, ref_grads, ref_xgrad):
    from pytorch_generative_b200 import losses

    xd = x.to(dev()).requires_grad_(True)
    m.zero_grad()
    logits = m(xd)
    loss = losses.bce_with_logits_sum_mean(logits, xd.detach())
    loss.backward()
    report = {"logits": _err(logits, ref_logits), "loss": _err(loss, ref_loss), "x grad": _err(xd.grad, ref_xgrad)}
    for k, p in m.named_parameters():
        report[k] = _err(p.grad, ref_grads[k])
    assert max(report.values()) <= TOL, report


def test_recipe_size_matches_oracle():
    state = _recipe_state()
    x = _binary((64, 1, 28, 28), 1)
    m = _model(dict(input_dim=784, hidden_dims=[8000]), state)
    logits, loss, grads, xgrad, after = R.loss_and_grads(state, x, 0)
    _check_step(m, x, logits, loss, grads, xgrad)
    for k, v in m.state_dict().items():
        if k in after:
            assert torch.equal(v.cpu(), after[k]), k


@pytest.mark.parametrize("name", ["one_hidden", "no_hidden", "two_hidden_three_masks"])
def test_fixture_forwards_match_the_reference(fixture, name):
    """Every forward of the fixture in sequence (four with n_masks=3): logits, loss and all gradients within the bf16
    tolerance; the masked weights and `mask` buffers exactly."""
    fx = fixture[name]
    m = _model(fx["kwargs"], fx["state_before"])
    for step in fx["forwards"]:
        _check_step(m, step["x"], step["logits"], step["loss"], step["grads"], step["x_grad"])
        sd = m.state_dict()
        for k, mask in step["masks"].items():
            assert torch.equal(sd[k].cpu(), mask.float()), k
    for k in fx["state_before"]:
        assert torch.equal(m.state_dict()[k].cpu(), fx["state_after"][k]), k
    assert m._mask_seed == len(fx["forwards"])


def test_autoregressive_property_is_exact():
    torch.manual_seed(3)
    from pytorch_generative_b200 import models

    m = models.MADE(64, [32, 48]).to(dev())
    order_pos = torch.from_numpy(m._connectivity(0)[0])  # sampling position of every dimension
    x = _binary((8, 64), 4).to(dev())
    with torch.no_grad():
        base = m(x)
        for t in (0, 1, 17, 40, 63):
            later = (order_pos >= t).to(dev())
            x2 = torch.where(later, 1.0 - x, x)
            out = m(x2)
            dims = (order_pos == t).nonzero()[0]
            assert torch.equal(out[:, dims], base[:, dims]), t


def test_fused_adam_trajectory_matches_oracle(fixture):
    from pytorch_generative_b200 import losses, optim

    fx = fixture["two_hidden_three_masks"]
    m = _model(fx["kwargs"], fx["state_before"])
    ref = R.TrainState(fx["state_before"], n_masks=3)
    opt = optim.FusedAdam(m.parameters())
    for s in range(3):
        x = _binary((16, 64), 10 + s)
        ref_loss, ref_norm = ref.step(x)
        xd = x.to(dev())
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(m(xd), xd)
        loss.backward()
        norm = opt.clip_and_step(1e50).item()
        assert abs(loss.item() - ref_loss) <= TOL * max(1.0, abs(ref_loss)), (s, loss.item(), ref_loss)
        assert abs(norm - ref_norm) <= 2.5e-2 * ref_norm, (s, norm, ref_norm)
    for k, p in m.named_parameters():
        assert _err(p, ref.p[k]) <= TOL, k


# --------------------------------------------------------------------------------------------------
# Sampling
# --------------------------------------------------------------------------------------------------
def _recorder():
    calls = []

    def fn(logits):
        calls.append(logits.detach().clone())
        return torch.zeros_like(logits)

    return calls, fn


@pytest.mark.parametrize("kwargs,n,tol", [(dict(input_dim=784, hidden_dims=[8000]), 16, 1e-3),
                                          (dict(input_dim=192, hidden_dims=[10]), 5, 1e-3),
                                          (dict(input_dim=64, hidden_dims=[32, 48], n_masks=3), 4, TOL),
                                          (dict(input_dim=64), 3, TOL)])
def test_teacher_forced_sampling_matches_full_forward(kwargs, n, tol):
    """Every entry given: sample_fn sees D calls of [n] logits in the reference's order, equal to the full forward's; the
    result is the input; a second call replays the captured step with the same logits."""
    from pytorch_generative_b200 import models

    torch.manual_seed(5)
    calls, fn = _recorder()
    m = models.MADE(**kwargs, sample_fn=fn).to(dev())
    D = kwargs["input_dim"]
    x = _binary((n, D), 6)
    runs = []
    for call in range(2):
        calls.clear()
        state = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}  # weights masked by earlier calls
        seed = m._mask_seed
        out = m.sample(conditioned_on=x.to(dev()))
        assert m._mask_seed == seed + 1
        assert torch.equal(out.cpu(), x)
        mask_set = seed % kwargs.get("n_masks", 1)
        order = np.argsort(R.connectivity(D, kwargs.get("hidden_dims") or [], mask_set)[-1])
        ref = R.forward(R.trainable(state), x, R.masks(R.connectivity(D, kwargs.get("hidden_dims") or [], mask_set)))
        assert len(calls) == D and all(c.shape == (n,) for c in calls)
        got = torch.stack([c.cpu() for c in calls], dim=1)
        assert _err(got, ref[:, order].detach()) <= tol, call
        runs.append(got)
    if kwargs.get("hidden_dims"):
        assert all(st["graph"] for st in m._made_sampler.values())
        if kwargs.get("n_masks", 1) == 1:
            assert torch.equal(runs[0], runs[1])


@pytest.mark.parametrize("name", ["one_hidden", "two_hidden_three_masks", "no_hidden"])
def test_sampling_under_predrawn_uniforms_matches_the_reference(fixture, name):
    """The reference's own samples, up to a knife-edge draw (|u - p| within the bf16 tolerance) and what follows it;
    given entries come back bit for bit."""
    fx = fixture[name]
    n_masks = fx["kwargs"].get("n_masks", 1)
    for kind in ("unconditional", "conditional"):
        s = fx[kind]
        from pytorch_generative_b200 import models

        m = models.MADE(**fx["kwargs"], sample_fn=R.uniform_sample_fn(s["uniforms"]))
        m.load_state_dict(fx["state_after"])  # with the _c/_h/_w of the reference's image forwards
        m = m.to(dev())
        m._mask_seed = s["mask_seed_before"]
        if s["conditioned_on"] is None:
            got = m.sample(s["sample"].shape[0]).cpu()
        else:
            got = m.sample(conditioned_on=s["conditioned_on"].to(dev())).cpu()
            given = s["conditioned_on"] >= 0
            assert torch.equal(got[given], s["conditioned_on"][given])
        ref = s["sample"]
        n = ref.shape[0]
        D = fx["kwargs"]["input_dim"]
        vecs = R.connectivity(D, fx["kwargs"].get("hidden_dims") or [], s["mask_seed_before"] % n_masks)
        order = np.argsort(vecs[-1])
        diff = (got.view(n, -1) != ref.view(n, -1))[:, order]
        if diff.any():
            first = int(diff.any(0).nonzero()[0])
            canvas = ref.view(n, -1).clone()
            canvas[:, order[first:]] = -1
            logits = R.forward(R.trainable(fx["state_after"]), canvas, R.masks(vecs))[:, order[first]]
            margin = (s["uniforms"][first] - torch.sigmoid(logits)).abs().min().item()
            assert margin < 2e-2, f"{kind}: samples diverge at step {first} without a knife-edge draw ({margin:.3e})"


# --------------------------------------------------------------------------------------------------
# Recipe
# --------------------------------------------------------------------------------------------------
def test_reproduce_made_trains_checkpoints_and_reloads(tmp_path):
    from pytorch_generative_b200 import models, recipes

    loader = [(_binary((64, 1, 28, 28), 20 + i).to(dev()), None) for i in range(2)]
    trainer = recipes.reproduce_made(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["optimizer"]["param_groups"][0]["lr"] == 1e-3 and "lr_scheduler" not in ckpt
    fresh = models.MADE(784, [8000])
    fresh.load_state_dict(ckpt["model"])
    for k, v in trainer.model.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v.cpu()), k
