"""NICE on the H100: the new kernels against float64 with per-element bounds, every GEMM stage of a training step against
float64 given the device's own bf16 inputs, the model against the reference's outputs (tests/golden/nice.pt) and against
the fp32 restatement at the recipe widths, invertibility, sampling, determinism, launch counts, a FusedAdam trajectory,
the step under a CUDA graph, the recipe, and deepcopy / pickle after sampling."""

import copy
import json
import os
import pickle

import pytest
import torch

import _gemm_reference as G
import _nice_reference as R
from _checks import check, check_equal

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nice.pt")
EPS = 2.0 ** -24  # fp32 unit roundoff
TOL = 1e-2        # bf16 GEMM operands, as the MADE tests: relative to max(1, max|ref|)
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
RECIPE = dict(n_features=784, n_coupling_blocks=4, n_hidden_layers=5, n_hidden_features=1000)


def dev():
    return torch.device("cuda:0")


def gamma(k):
    return k * EPS / (1 - k * EPS)


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _err(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _loaded(kwargs, state):
    from pytorch_generative_b200 import models

    m = models.NICE(**kwargs)
    m.load_state_dict(state)
    return m.to(dev())


def _model(kwargs, seed):
    """NICE under `seed`, log-scales spread by N(0, 0.1) so that the scaling is not the identity, on the GPU."""
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = models.NICE(**kwargs)
    with torch.no_grad():
        m.scaling.log_scale.normal_(0, 0.1)
    return m.to(dev())


def _dequantized(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(0, 256, shape, generator=g).float() + torch.rand(shape, generator=g)) / 256


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev())


# --------------------------------------------------------------------------------------------------
# kernels
# --------------------------------------------------------------------------------------------------
KERNEL_CASES = [(n, D) for D in (2, 30, 784, 3072) for n in (1, 5, 1024)]


@pytest.mark.parametrize("n, D", KERNEL_CASES)
def test_split_and_join_against_float64(n, D):
    """Without scaling both are exact copies; with it each entry is within 4 ulp of x * exp(+-s) (expf's 2 ulp, the
    product's rounding and a spare).  Pad columns of the halves, NaN before the launch, come out zero; the bf16 copy is bf16 of
    the half.  log_det is one ascending fp32 chain: within gamma(D) sum |s|."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(n * 7 + D)
    x = torch.randn(n, D, generator=g).to(dev())
    s = (torch.randn(1, D, generator=g) * 0.5).to(dev())
    h_lo, h_hi, ld = D // 2, D - D // 2, (D - D // 2 + 7) // 8 * 8
    for scale, sign in ((None, 1.0), (s, 1.0), (s, -1.0)):
        for half in (0, 1):
            lo, hi, xb = _nan((n, ld), F32), _nan((n, ld), F32), _nan((n, ld), BF16)
            L.nice_split(x, lo, hi, scale, sign, out_bf16=xb, bf16_half=half)
            ref = x.to(F64) if scale is None else x.to(F64) * torch.exp(sign * s.to(F64))
            bound = torch.zeros_like(ref) if scale is None else 8 * EPS * ref.abs()
            check("split lo", lo[:, :h_lo], ref[:, :h_lo], bound[:, :h_lo])
            check("split hi", hi[:, :h_hi], ref[:, h_lo:], bound[:, h_lo:])
            for name, buf, w in (("lo", lo, h_lo), ("hi", hi, h_hi)):
                assert bool((buf[:, w:] == 0).all()), f"{name} pads"
            check_equal("split bf16", xb, (hi if half else lo).to(BF16))
        z = _nan((n, D), F32)
        log_det = _nan((), F32)
        L.nice_join(lo, hi, z, scale, sign, log_det=None if scale is None else log_det)
        src = torch.cat((lo[:, :h_lo], hi[:, :h_hi]), 1).to(F64)
        ref = src if scale is None else src * torch.exp(sign * s.to(F64))
        check("join", z, ref, torch.zeros_like(ref) if scale is None else 8 * EPS * ref.abs())
        if scale is not None:
            s64 = s.to(F64)
            check("log_det", log_det.view(1), s64.sum().view(1), (gamma(D) * s64.abs().sum()).view(1))


@pytest.mark.parametrize("n, D", KERNEL_CASES)
def test_scale_backward_against_float64(n, D):
    """d_lo, d_hi = dz exp(s) within 4 ulp, their bf16 copy, pads zero; d_log_scale = g + sum_b dz z: batch slices of up
    to 128 images (one fmaf chain each) added in slice order after g, within gamma(n + 2) (sum |dz z| + |g|)."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(n * 11 + D)
    dz, z = torch.randn(n, D, generator=g).to(dev()), torch.randn(n, D, generator=g).to(dev())
    s = (torch.randn(1, D, generator=g) * 0.5).to(dev())
    g_ld = torch.tensor(0.75, device=dev())
    h_lo, h_hi, ld = D // 2, D - D // 2, (D - D // 2 + 7) // 8 * 8
    for half in (0, 1):
        d_lo, d_hi, dm, ds = _nan((n, ld), F32), _nan((n, ld), F32), _nan((n, ld), BF16), _nan((1, D), F32)
        L.nice_scale_bwd(dz, z, s, g_ld, d_lo, d_hi, ds, dm_bf16=dm, bf16_half=half)
        ref = dz.to(F64) * torch.exp(s.to(F64))
        check("d_lo", d_lo[:, :h_lo], ref[:, :h_lo], 8 * EPS * ref[:, :h_lo].abs())
        check("d_hi", d_hi[:, :h_hi], ref[:, h_lo:], 8 * EPS * ref[:, h_lo:].abs())
        assert bool((d_lo[:, h_lo:] == 0).all()) and bool((d_hi[:, h_hi:] == 0).all())
        check_equal("dm", dm, (d_hi if half else d_lo).to(BF16))
        prod = dz.to(F64) * z.to(F64)
        ref_s = prod.sum(0, keepdim=True) + 0.75
        check("d_log_scale", ds, ref_s, gamma(n + 2) * (prod.abs().sum(0, keepdim=True) + 0.75))
    ds = _nan((1, D), F32)  # no images: d_log_scale = g
    L.nice_scale_bwd(dz[:0], z[:0], s, g_ld, d_lo[:0], d_hi[:0], ds)
    assert bool((ds == 0.75).all())


@pytest.mark.parametrize("n, D", KERNEL_CASES)
def test_logistic_prior_against_float64(n, D):
    """log_prob[b] = -sum_j |z| + 2 log1p(exp(-|z|)): every term is within a few ulp (expf, log1pf, two roundings) and
    the row sum adds at most D - 1 roundings, so within gamma(D + 8) of the sum of the (positive) terms; dz =
    scale tanh(z / 2) within 4 ulp (tanhf's 2 and a spare)."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(n * 13 + D)
    z = (torch.randn(n, D, generator=g) * 3).to(dev())
    log_prob, dz = _nan((n,), F32), _nan((n, D), F32)
    L.logistic_prior_fwd_bwd(z, log_prob, dz, grad_scale=-0.5)
    z64 = z.to(F64)
    terms = torch.nn.functional.softplus(z64) + torch.nn.functional.softplus(-z64)
    check("log_prob", log_prob, -terms.sum(1), gamma(D + 8) * terms.sum(1))
    ref = -0.5 * torch.tanh(z64 / 2)
    check("dz", dz, ref, 8 * EPS * ref.abs() + 1e-45)


# --------------------------------------------------------------------------------------------------
# every GEMM stage of a training step, given the device's own bf16 inputs
# --------------------------------------------------------------------------------------------------
def _record_gemms(monkeypatch):
    """Wraps _lib.gemm so that every launch's operands, epilogue inputs and outputs are kept (cloned around the call)."""
    from pytorch_generative_b200 import _lib as L

    calls, orig = [], L.gemm

    def gemm(A, B, M, N, K, **kw):
        rec = dict(A=A.clone(), B=B.clone(), M=M, N=N, K=K,
                   kw={k: v.clone() if torch.is_tensor(v) else v for k, v in kw.items()})
        orig(A, B, M, N, K, **kw)
        rec["out"] = {k: kw[k].clone() for k in ("out_f32", "out_bf16", "out_pre", "bias_grad")
                      if kw.get(k) is not None}
        calls.append(rec)

    monkeypatch.setattr(L, "gemm", gemm)
    return calls


def _replay(i, rec):
    """One GEMM launch against float64: acc = A B^T on the logical operands, t = alpha acc + bias, times relu'(aux)
    when dact is ReLU-from-output, pre = t + res0 (+ c0 when accumulating).  fp32 outputs within the GEMM bound with
    the bias, residual and c0 magnitudes joining the terms and three more roundings; bf16 outputs add bf16's half ulp."""
    from pytorch_generative_b200 import _lib as L

    kw, M, N, K = rec["kw"], rec["M"], rec["N"], rec["K"]
    A = (rec["A"].t() if kw.get("a_mn") else rec["A"])[:M, :K].to(F64)
    B = (rec["B"].t() if kw.get("b_mn") else rec["B"])[:N, :K].to(F64)
    alpha = kw.get("alpha", 1.0)
    t = alpha * (A @ B.t())
    mag = abs(alpha) * (A.abs() @ B.abs().t())
    if kw.get("bias") is not None:
        t = t + kw["bias"][:N].to(F64)
        mag = mag + kw["bias"][:N].to(F64).abs()
    if kw.get("dact", L.ACT_NONE) == L.ACT_RELU_OUT:
        keep = (kw["aux"][:M, :N].float() > 0).to(F64)
        t, mag = t * keep, mag * keep
    if kw.get("res0") is not None:
        t = t + kw["res0"][:M, :N].to(F64)
        mag = mag + kw["res0"][:M, :N].to(F64).abs()
    c0 = kw["out_f32"][:M, :N] if kw.get("accumulate") else None
    if c0 is not None:
        t = t + c0.to(F64)
    b32 = G.bound(K + 3, 1.0, mag, c0, kw.get("split_k", 1))
    name = f"gemm {i} ({M}x{N}x{K}, a_mn={kw.get('a_mn', False)}, b_mn={kw.get('b_mn', False)})"
    out = rec["out"]
    if "out_f32" in out:
        check(name + " out_f32", out["out_f32"][:M, :N], t, b32)
    if "out_pre" in out:
        check(name + " out_pre", out["out_pre"][:M, :N], t, b32 + 2.0 ** -8 * (t.abs() + b32))
    if "out_bf16" in out:
        act = torch.relu(t) if kw.get("act", 0) & 0xFF == L.ACT_RELU else t
        check(name + " out_bf16", out["out_bf16"][:M, :N], act, b32 + 2.0 ** -8 * (act.abs() + b32))
    if "bias_grad" in out:
        d0 = kw["bias_grad"][:M]
        check(name + " bias_grad", out["bias_grad"][:M], d0.to(F64) + A.sum(1),
              G.rowsum_bound(K, A.abs().sum(1), d0, kw.get("split_k", 1)))


@pytest.mark.parametrize("kwargs, n", [(RECIPE, 64), (dict(n_features=30, n_coupling_blocks=3, n_hidden_layers=2,
                                                            n_hidden_features=20), 37)])
def test_every_gemm_stage_of_a_training_step_against_float64(monkeypatch, kwargs, n):
    from pytorch_generative_b200 import losses

    m = _model(kwargs, seed=3)
    x = _dequantized((n, kwargs["n_features"]), seed=4).to(dev()).requires_grad_(True)
    calls = _record_gemms(monkeypatch)
    losses.logistic_prior_nll(x, None, m(x))["loss"].backward()
    torch.cuda.synchronize()
    L_ = kwargs["n_hidden_layers"] + 1
    B = kwargs["n_coupling_blocks"]
    assert len(calls) == B * L_ + B * (2 * L_), len(calls)  # forward; wgrad and dgrad per layer
    for i, rec in enumerate(calls):
        _replay(i, rec)


# --------------------------------------------------------------------------------------------------
# end to end
# --------------------------------------------------------------------------------------------------
def test_the_reference_outputs(fixture):
    """z, log_det_J, the loss dict, every gradient, the input gradient and _inverse(z) of the reference at 1e-2."""
    from pytorch_generative_b200 import losses

    for name, fx in fixture.items():
        m = _loaded(fx["kwargs"], fx["state"])
        x = fx["x"].to(dev()).requires_grad_(True)
        z, log_det = m(x)
        assert z.shape == x.shape and log_det.dim() == 0
        out = losses.logistic_prior_nll(x, None, (z, log_det))
        out["loss"].backward()
        assert _err(z, fx["z"]) <= TOL and _err(log_det, fx["log_det_J"]) <= TOL, name
        for k, v in fx["losses"].items():
            assert _err(out[k], v) <= TOL, (name, k)
        for k, prm in m.named_parameters():
            assert _err(prm.grad, fx["grads"][k]) <= TOL, (name, k)
        assert _err(x.grad, fx["x_grad"]) <= TOL, name
        with torch.no_grad():
            assert _err(m._inverse(fx["z"].to(dev())), fx["inverse"]) <= TOL, name
            assert torch.equal(m._forward(x), z)


def test_recipe_widths_against_the_fp32_restatement():
    from pytorch_generative_b200 import losses

    m = _model(RECIPE, seed=5)
    state = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    x = _dequantized((64, 1, 28, 28), seed=6)
    rz, rld, rloss, rgrads, rxg = R.loss_and_grads(state, x, F32, dev())
    xd = x.to(dev()).requires_grad_(True)
    z, log_det = m(xd)
    out = losses.logistic_prior_nll(xd, None, (z, log_det))
    out["loss"].backward()
    assert _err(z, rz) <= TOL and _err(log_det, rld) <= TOL
    for k, v in rloss.items():
        assert _err(out[k], v) <= TOL, k
    for k, prm in m.named_parameters():
        assert _err(prm.grad, rgrads[k]) <= TOL, k
    assert _err(xd.grad, rxg) <= TOL


def test_standalone_modules_match_the_restatement():
    """AdditiveCouplingBlock and ScalingLayer run on their own on the same kernels, with gradients."""
    m = _model(dict(n_features=30, n_coupling_blocks=2, n_hidden_layers=2, n_hidden_features=20), seed=7)
    params = {k: v.detach().to(F64) for k, v in m.state_dict().items()}
    x = torch.randn(9, 30, device=dev(), requires_grad=True)
    for b, block in enumerate(m.net):
        y = block(x)
        assert _err(y, R.couple(params, b, x.detach().to(F64), 1)) <= TOL
        y.sum().backward()
    z = m.scaling(x.view(9, 3, 10))
    assert z.shape == (9, 3, 10)
    assert _err(z.view(9, 30), x.detach().to(F64) * torch.exp(params["scaling.log_scale"])) <= 1e-5
    ld = m.scaling.log_det_J()
    assert ld.dim() == 0 and _err(ld, params["scaling.log_scale"].sum()) <= 1e-5
    (z.sum() + ld).backward()
    assert m.scaling.log_scale.grad is not None and x.grad is not None


# --------------------------------------------------------------------------------------------------
# invertibility
# --------------------------------------------------------------------------------------------------
def test_coupling_block_round_trip():
    """Per block: the pass-through half is returned bit for bit, the inverse reproduces m bit for bit (the same bf16
    operand through the same GEMMs; alpha = -1 and the negated bias give exactly -fl(acc + b)), and the transformed half
    is within 2^-23 (|x2| + |m|): two roundings of the add and the subtract."""
    m = _model(RECIPE, seed=8)
    x = _dequantized((64, 784), seed=9).to(dev())
    with torch.no_grad():
        for block in m.net:
            c, t = (slice(392, None), slice(0, 392)) if block.reverse else (slice(0, 392), slice(392, None))
            y = block(x)
            back = block.inverse(y)
            check_equal("pass-through", y[:, c], x[:, c])
            check_equal("pass-through back", back[:, c], x[:, c])
            probe = x.clone()
            probe[:, t] = 0
            mm = block(probe)[:, t]                  # 0 + m = m exactly
            check_equal("m", block.inverse(probe)[:, t], -mm)  # 0 - m
            bound = 2.0 ** -23 * (x[:, t].to(F64).abs() + mm.to(F64).abs())
            check("transformed half", back[:, t], x[:, t], bound)
            x = y


def test_scaling_round_trip():
    m = _model(dict(n_features=30, n_coupling_blocks=2, n_hidden_layers=1, n_hidden_features=8), seed=10)
    x = torch.randn(17, 30, device=dev())
    with torch.no_grad():
        back = m.scaling.inverse(m.scaling(x))
    check("scaling round trip", back, x, 16 * EPS * x.to(F64).abs())


def test_whole_model_round_trip():
    """inverse(forward(x)) is within 1e-2 of max(1, |x|).  This is looser than the block round trip: the scaling's
    round trip can be an ulp off, and an ulp in a conditioning half can flip the bf16 operand of the next coupling MLP,
    whose m then differs by a bf16-sized step."""
    m = _model(RECIPE, seed=11)
    x = _dequantized((128, 1, 28, 28), seed=12).to(dev())
    with torch.no_grad():
        z, _ = m(x)
        back = m._inverse(z)
    check("round trip", back, x, 1e-2 * x.to(F64).abs().clamp_min(1.0))


def test_the_inverse_is_inference_only():
    m = _model(dict(n_features=8, n_coupling_blocks=2, n_hidden_layers=1, n_hidden_features=8), seed=13)
    z = torch.randn(3, 8, device=dev())
    for call in (lambda: m._inverse(z), lambda: m.net[0].inverse(z), lambda: m.scaling.inverse(z)):
        with pytest.raises(RuntimeError, match="inference-only"):
            call()


def test_other_dtypes_raise_instead_of_launching():
    from pytorch_generative_b200 import _lib as L

    for cast in (lambda m: m.double(), lambda m: m.half()):
        m = cast(_model(dict(n_features=8, n_coupling_blocks=2, n_hidden_layers=1, n_hidden_features=8), seed=14))
        before = L.launch_count()
        with pytest.raises(RuntimeError, match="fp32"):
            m(torch.randn(3, 8, device=dev()))
        assert L.launch_count() == before


# --------------------------------------------------------------------------------------------------
# sampling and determinism
# --------------------------------------------------------------------------------------------------
def test_sample_is_the_inverse_of_the_reference_latents(fixture):
    for name, fx in fixture.items():
        m = _loaded(fx["kwargs"], fx["state_after"])
        torch.manual_seed(fx["sample_seed"])
        got = m.sample(fx["x"].shape[0], temp=0.7)
        torch.manual_seed(fx["sample_seed"])
        latents = torch.randn(fx["x"].shape) * 0.7
        with torch.no_grad():
            check_equal(name, got, m._inverse(latents.to(dev())))
        assert _err(got, fx["sample"]) <= TOL, name
        # deepcopy and pickle after sample()
        clone = copy.deepcopy(m)
        again = pickle.loads(pickle.dumps(m))
        for other in (clone, again):
            torch.manual_seed(fx["sample_seed"])
            check_equal(name + " copy", other.sample(fx["x"].shape[0], temp=0.7), got)


def test_repeat_runs_and_sub_batches_are_bit_identical():
    from pytorch_generative_b200 import losses

    m = _model(RECIPE, seed=15)
    x = _dequantized((96, 1, 28, 28), seed=16).to(dev())
    runs = []
    for _ in range(2):
        m.zero_grad()
        z, log_det = m(x)
        losses.logistic_prior_nll(x, None, (z, log_det))["loss"].backward()
        runs.append((z.detach().clone(), log_det.detach().clone(), [p.grad.clone() for p in m.parameters()]))
    check_equal("z", runs[0][0], runs[1][0])
    check_equal("log_det", runs[0][1], runs[1][1])
    for a, b in zip(runs[0][2], runs[1][2]):
        check_equal("grad", a, b)
    with torch.no_grad():
        check_equal("sub-batch", m(x[17:40])[0], runs[0][0][17:40])
        check_equal("inverse sub-batch", m._inverse(runs[0][0][17:40]), m._inverse(runs[0][0])[17:40])


def test_launch_count():
    """Forward: split, B L GEMMs, join = B L + 2.  Loss: 1.  Backward: the scaling's backward and its partial sum (2),
    per block L wgrads and L dgrads (block 0's first-layer dgrad only with an input gradient), the final join with an
    input gradient, and 2 partial sums per weight-gradient GEMM that runs split-K (its tile slices and its bias sums)."""
    from pytorch_generative_b200 import _lib as L, losses, ops

    kwargs = RECIPE
    B, Lyr = kwargs["n_coupling_blocks"], kwargs["n_hidden_layers"] + 1
    m = _model(kwargs, seed=17)
    for n, input_grad in ((64, False), (1024, True)):
        x = _dequantized((n, 784), seed=18).to(dev()).requires_grad_(input_grad)
        widths = [784 // 2] + [kwargs["n_hidden_features"]] * (Lyr - 1) + [784 // 2]
        split_sums = sum(2 for i in range(Lyr) if ops._split_k_for(ops.round_up(widths[i + 1], 8),
                                                                    ops.round_up(widths[i], 8), n) > 1)
        out = losses.logistic_prior_nll(x, None, m(x))  # warm-up
        out["loss"].backward()
        torch.cuda.synchronize()
        before = L.launch_count()
        z, log_det = m(x)
        fwd = L.launch_count() - before
        out = losses.logistic_prior_nll(x, None, (z, log_det))
        out["loss"].backward()
        total = L.launch_count() - before
        assert fwd == B * Lyr + 2
        expected = fwd + 1 + 2 + B * 2 * Lyr - (0 if input_grad else 1) + int(input_grad) + B * split_sums
        assert total == expected, (n, total, expected)


# --------------------------------------------------------------------------------------------------
# training
# --------------------------------------------------------------------------------------------------
def test_fused_adam_trajectory_matches_the_restatement(fixture):
    from pytorch_generative_b200 import losses, optim

    fx = fixture["nice_64"]
    m = _loaded(fx["kwargs"], fx["state"])
    params = {k: v.clone().requires_grad_(True) for k, v in R.params_of(fx["state"]).items()}
    ref_opt = torch.optim.Adam([params[k] for k in R.names(fx["state"])], lr=1e-3)
    opt = optim.FusedAdam(m.parameters(), lr=1e-3)
    for s in range(3):
        x = _dequantized((16, 1, 8, 8), seed=20 + s)
        ref_opt.zero_grad()
        ref_loss = R.loss(*R.forward(params, x))["loss"]
        ref_loss.backward()
        ref_norm = torch.nn.utils.clip_grad_norm_(list(params.values()), 1e50).item()
        ref_opt.step()
        xd = x.to(dev())
        opt.zero_grad()
        loss = losses.logistic_prior_nll(xd, None, m(xd))["loss"]
        loss.backward()
        norm = opt.clip_and_step(1e50).item()
        assert abs(loss.item() - ref_loss.item()) <= TOL * max(1.0, abs(ref_loss.item())), s
        assert abs(norm - ref_norm) <= TOL * ref_norm, (s, norm, ref_norm)
    for k, prm in m.named_parameters():
        assert _err(prm, params[k]) <= TOL, k


class _Preds(tuple):
    """(z, log_det_J) with the .detach() that GraphedTrainStep applies to a model's output."""

    def detach(self):
        return _Preds(t.detach() for t in self)


class _TupleModel(torch.nn.Module):
    def __init__(self, nice):
        super().__init__()
        self.nice = nice

    def forward(self, x):
        return _Preds(self.nice(x))


def _tuple_loss(preds, x):
    from pytorch_generative_b200 import losses

    return losses.logistic_prior_nll(x, None, preds)["loss"]


def test_graphed_train_step_equals_the_eager_step():
    """The forward and backward never synchronise with the host, so the step captures as a CUDA graph; two replays
    equal two eager steps bit for bit."""
    from pytorch_generative_b200 import trainstep

    kwargs = dict(n_features=784, n_coupling_blocks=4, n_hidden_layers=2, n_hidden_features=256)
    init = _model(kwargs, seed=21)
    state = {k: v.clone() for k, v in init.state_dict().items()}
    xs = [_dequantized((128, 1, 28, 28), seed=22 + s).to(dev()) for s in range(2)]
    graphed = _TupleModel(copy.deepcopy(init))
    step = trainstep.GraphedTrainStep(graphed, graphed.parameters(), _tuple_loss, xs[0], lr=1e-3, lr_gamma=1.0)
    step.reset({f"nice.{k}": v for k, v in state.items()}, lr=1e-3)
    eager = _TupleModel(copy.deepcopy(init))
    eager.nice.load_state_dict(state)
    params = list(eager.parameters())
    opt = torch.optim.Adam(params, lr=torch.tensor(1e-3, device=dev()), capturable=True)
    for x in xs:
        loss_g, norm_g = step(x)
        opt.zero_grad(set_to_none=True)
        loss = _tuple_loss(eager(x), x)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(params, 1e50, foreach=True)
        opt.step()
        assert loss_g == loss.item() and norm_g == norm.item()
    for (k, a), b in zip(graphed.named_parameters(), params):
        check_equal(k, a.detach(), b.detach())


def test_reproduce_nice_trains_logs_checkpoints_and_samples(tmp_path, capsys):
    from pytorch_generative_b200 import models, recipes

    loader = [(_dequantized((64, 1, 28, 28), seed=30 + i).to(dev()), None) for i in range(2)]
    trainer = recipes.reproduce_nice(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["optimizer"]["param_groups"][0]["lr"] == 1e-3 and "lr_scheduler" not in ckpt
    fresh = models.NICE(784)
    fresh._register_shape(1, 28, 28)
    assert list(ckpt["model"]) == list(fresh.state_dict())
    # the layout of the reference's own state dicts: the image-shape buffers, then the blocks, then the scaling
    for fx in torch.load(GOLD, weights_only=False).values():
        assert [k.split(".")[0] for k in fx["state_after"]][:3] == [k.split(".")[0] for k in ckpt["model"]][:3]
        assert list(fx["state_after"])[-1] == list(ckpt["model"])[-1] == "scaling.log_scale"
    fresh.load_state_dict(ckpt["model"])
    for k, v in trainer.model.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v.cpu()), k
    tags = set()
    with open(tmp_path / "metrics.jsonl") as f:
        for line in f:
            tags.add(json.loads(line)["tag"])
    for key in ("loss", "prior_log_likelihood", "log_det_J", "grad_norm"):
        assert f"metrics/{key}" in tags, key
    capsys.readouterr()
    trainer.sample_one_batch()
    assert "Failed to sample" not in capsys.readouterr().out
    assert bool(torch.isfinite(trainer.model.sample(16)).all())
