"""AdaBelief (pg_adabelief_step, optim.AdaBelief) and ReZero (pg_rezero_fwd / _bwd, nn.ReZeroWrapper) on the GPU:
the kernels against float64 restatements with per-element bounds (tests/_adabelief_reference.py), the optimizer and the
module against the reference's fixture (tests/golden/adabelief_rezero.pt), the Trainer, determinism and CUDA graphs."""

import math
import os

import pytest
import torch

import _adabelief_reference as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "adabelief_rezero.pt")
DEV = torch.device("cuda")


@pytest.fixture(scope="module")
def fx():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return torch.load(GOLD, weights_only=False)


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements out of bound, worst {float((err - bound).max()):.3e}"


# ----------------------------------------------------------------------------------------------------------------------
# pg_adabelief_step
# ----------------------------------------------------------------------------------------------------------------------
NUMELS = (1, 3, 4, 4097, 65536 + 5, 3 * 65536 + 17)
MISALIGNED = ((4097, 1), (5, 3))  # (numel, offset in floats): views that take the scalar path


def _tensors(seed):
    """p, g, m, v lists on the device: NUMELS as whole tensors, MISALIGNED as views at an odd offset."""
    g = torch.Generator().manual_seed(seed)
    out = [[], [], [], []]
    shapes = [(n, 0) for n in NUMELS] + list(MISALIGNED)
    for n, off in shapes:
        vals = (torch.randn(n, generator=g), torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.1,
                torch.rand(n, generator=g) * 0.01)
        for lst, v in zip(out, vals):
            buf = torch.empty(n + off, device=DEV)
            t = buf[off:]
            t.copy_(v)
            lst.append(t)
    return out


def _raw_step(ps, gs, ms, vs, max_norm, skip_above, lr, beta1, beta2, step):
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200 import optim

    numel, chunks, n_chunks = optim.chunk_table([p.numel() for p in ps], DEV)
    ptrs = torch.tensor([[t.data_ptr() for t in row] for row in (ps, gs, ms, vs)], dtype=torch.int64, device=DEV)
    partials = torch.empty(n_chunks, device=DEV)
    norm_out = torch.zeros(2, device=DEV)
    L.grad_sqnorm(ptrs[1], numel, chunks, n_chunks, optim.CHUNK, partials)
    L.adabelief_step(ptrs[0], ptrs[1], ptrs[2], ptrs[3], numel, chunks, n_chunks, optim.CHUNK, partials, n_chunks,
                     max_norm, skip_above, lr, beta1, beta2, step, norm_out)
    torch.cuda.synchronize()
    return norm_out.cpu(), n_chunks


@pytest.mark.parametrize("step", [1, 2, 1000])
@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.8, 0.99)])
@pytest.mark.parametrize("clip", [False, True])
def test_adabelief_step_kernel_against_float64(fx, step, betas, clip):
    ps, gs, ms, vs = _tensors(step + int(clip))
    before = [[t.clone() for t in lst] for lst in (ps, gs, ms, vs)]
    total = math.sqrt(sum(float(g.double().pow(2).sum()) for g in gs))
    max_norm = 0.3 * total if clip else 3.0e38
    lr = 2e-3
    norm_out, n_chunks = _raw_step(ps, gs, ms, vs, max_norm, 0.0, lr, *betas, step)
    ref_norm, b_norm = R.sqnorm_reference(before[1], n_chunks)
    assert abs(float(norm_out[0]) - ref_norm) <= b_norm and float(norm_out[1]) == 1.0
    sc = R.scalars(lr, *betas, step)
    for i in range(len(ps)):
        ref = R.reference(before[0][i], before[1][i], before[2][i], before[3][i], float(norm_out[0]), max_norm, sc)
        for key, got in (("p", ps[i]), ("g", gs[i]), ("m", ms[i]), ("v", vs[i])):
            _within(got, ref[key], ref["b_" + key], f"{key}[{ps[i].numel()}]")
        if not clip:
            assert torch.equal(gs[i], before[1][i]), "an unclipped step wrote the gradient"


@pytest.mark.parametrize("side", ["below", "above"])
def test_adabelief_skip_rule(fx, side):
    ps, gs, ms, vs = _tensors(5)
    before = [[t.clone() for t in lst] for lst in (ps, gs, ms, vs)]
    total = math.sqrt(sum(float(g.double().pow(2).sum()) for g in gs))
    skip_above = total * (1.01 if side == "below" else 0.99)
    norm_out, _ = _raw_step(ps, gs, ms, vs, 3.0e38, skip_above, 1e-3, 0.9, 0.999, 1)
    applied = [not torch.equal(a, b) for a, b in zip(ps, before[0])]
    if side == "below":
        assert float(norm_out[1]) == 1.0 and all(applied)
    else:
        assert float(norm_out[1]) == 0.0
        for lst, old in zip((ps, gs, ms, vs), before):
            assert all(torch.equal(a, b) for a, b in zip(lst, old))


@pytest.mark.parametrize("skip", [True, False])
def test_adabelief_nan_norm(fx, skip):
    ps, gs, ms, vs = _tensors(6)
    gs[3][7] = float("nan")
    before = [[t.clone() for t in lst] for lst in (ps, gs, ms, vs)]
    norm_out, _ = _raw_step(ps, gs, ms, vs, 1.0, 1e30 if skip else 0.0, 1e-3, 0.9, 0.999, 1)
    assert math.isnan(float(norm_out[0]))
    if skip:
        assert float(norm_out[1]) == 0.0
        for lst, old in zip((ps, gs, ms, vs), before):
            assert all(_same_bits(a, b) for a, b in zip(lst, old))
        return
    # clip_grad_norm_ followed by the step: every gradient, moment and parameter becomes NaN
    leaves = [torch.nn.Parameter(p.clone()) for p in before[0]]
    for leaf, g in zip(leaves, before[1]):
        leaf.grad = g.clone()
    assert math.isnan(float(torch.nn.utils.clip_grad_norm_(leaves, 1.0)))
    sc = R.scalars(1e-3, 0.9, 0.999, 1)
    for i in range(len(ps)):
        ref = R.reference(before[0][i], leaves[i].grad, before[2][i], before[3][i], float("nan"), 1.0, sc)
        for key, got in (("p", ps[i]), ("g", gs[i]), ("m", ms[i]), ("v", vs[i])):
            assert bool(torch.isnan(got).all()) and bool(torch.isnan(ref[key]).all()), key


# ----------------------------------------------------------------------------------------------------------------------
# optim.AdaBelief against the reference's trajectory
# ----------------------------------------------------------------------------------------------------------------------
def _setup(init=None):
    from pytorch_generative_b200.optim import AdaBelief

    init = init or R.initial_params()
    params = {k: torch.nn.Parameter(v.clone().to(DEV)) for k, v in init.items()}
    groups = [dict(params=[params[n] for n in gr["names"]], lr=gr["lr"], betas=gr["betas"]) for gr in R.GROUPS]
    return params, AdaBelief(groups)


def _run_steps(params, opt, first, last):
    from pytorch_generative_b200 import _lib as L

    launches = []
    for t in range(first, last + 1):
        grads = R.grads_at(t)
        for k, p in params.items():
            p.grad = None if grads[k] is None else grads[k].to(DEV)
        max_norm = float("inf")
        if t in R.CLIP_STEPS:
            max_norm = R.CLIP_FRACTION * float(torch.linalg.vector_norm(torch.cat([g for g in grads.values() if g is not None])))
        n0 = L.launch_count()
        opt.clip_and_step(max_norm)
        launches.append(L.launch_count() - n0)
    torch.cuda.synchronize()
    return launches


def _compare_to_fixture(fx, params, opt, t):
    rec = fx["adabelief"]["steps"][t - 1]
    for k in rec["p"]:
        st = opt.state[params[k]]
        assert type(st["step"]) is int and st["step"] == rec["step"][k]
        for key, got in (("p", params[k].detach()), ("m", st["ema_avg"]), ("v", st["ema_var"])):
            got = got.cpu()
            ref = R.unpack(rec[key][k])
            tol = 1e-5 * max(1.0, float(ref.abs().max()))
            assert float((got - ref).abs().max()) <= tol, (t, k, key)


def test_optimizer_follows_the_reference_trajectory(fx):
    params, opt = _setup()
    for t in range(1, R.STEPS + 1):
        launches = _run_steps(params, opt, t, t)
        assert launches == [3], "one norm launch plus one launch per group"
        _compare_to_fixture(fx, params, opt, t)
    assert params["none"] not in opt.state or not opt.state[params["none"]]
    assert torch.equal(params["none"].detach().cpu(), R.initial_params()["none"])


def test_optimizer_continues_from_a_reference_state_dict(fx):
    sd = fx["adabelief"]["state_dicts"]
    params, opt = _setup({k: R.unpack(v) for k, v in sd["params_3"].items()})
    opt.load_state_dict(R.unpack_state_dict(sd[3]))
    for t in range(4, R.STEPS + 1):
        _run_steps(params, opt, t, t)
        _compare_to_fixture(fx, params, opt, t)


def test_optimizer_is_deterministic_and_keeps_the_reference_layout(fx):
    runs = []
    for _ in range(2):
        params, opt = _setup()
        _run_steps(params, opt, 1, R.STEPS)
        runs.append((params, opt))
    (pa, oa), (pb, ob) = runs
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k
        if k != "none":
            for n in ("ema_avg", "ema_var"):
                assert torch.equal(oa.state[pa[k]][n], ob.state[pb[k]][n])
    ref_sd, sd = fx["adabelief"]["state_dicts"][3], oa.state_dict()
    assert [set(g) for g in sd["param_groups"]] == [set(g) for g in ref_sd["param_groups"]]
    assert sorted(sd["state"]) == sorted(ref_sd["state"])
    for i, st in sd["state"].items():
        assert list(st) == ["step", "ema_avg", "ema_var"] and type(st["step"]) is int


def test_skipped_first_step_creates_no_state(fx):
    from pytorch_generative_b200.optim import AdaBelief

    p = torch.nn.Parameter(torch.randn(100, device=DEV))
    p.grad = torch.randn(100, device=DEV)
    opt = AdaBelief([p])
    before = p.detach().clone()
    empty = opt.state_dict()
    opt.clip_and_step(skip_above=1e-3)
    assert torch.equal(p.detach(), before) and p not in opt.state
    assert opt.state_dict() == empty
    opt.clip_and_step(skip_above=1e9)  # the next step creates state and applies
    assert opt.state[p]["step"] == 1 and not torch.equal(p.detach(), before)


def test_multiplicative_lr_between_steps(fx):
    from pytorch_generative_b200.optim import AdaBelief

    g = torch.Generator().manual_seed(9)
    p = torch.nn.Parameter(torch.randn(5000, generator=g).to(DEV))
    opt = AdaBelief([p], lr=1e-2, betas=(0.85, 0.995))
    sched = torch.optim.lr_scheduler.MultiplicativeLR(opt, lr_lambda=lambda _: 0.5)
    for t in range(1, 4):
        p.grad = torch.randn(5000, generator=g).to(DEV)
        st = opt.state.get(p)
        m0 = st["ema_avg"].clone() if st else torch.zeros_like(p)
        v0 = st["ema_var"].clone() if st else torch.zeros_like(p)
        p0, g0, lr = p.detach().clone(), p.grad.clone(), opt.param_groups[0]["lr"]
        norm = opt.clip_and_step()
        ref = R.reference(p0, g0, m0, v0, float(norm), 3.0e38, R.scalars(lr, 0.85, 0.995, t))
        _within(p.detach(), ref["p"], ref["b_p"], f"p at step {t}")
        sched.step()
    assert abs(opt.param_groups[0]["lr"] - 1e-2 / 8) < 1e-15


# ----------------------------------------------------------------------------------------------------------------------
# the Trainer with AdaBelief
# ----------------------------------------------------------------------------------------------------------------------
def _trainer(tmp_path, seed=0):
    from pytorch_generative_b200 import models, optim, recipes, trainer

    torch.manual_seed(seed)
    m = models.PixelCNN(in_channels=1, out_channels=1, n_residual=1, residual_channels=16, head_channels=16)
    opt = optim.AdaBelief(m.parameters(), lr=2e-3)
    g = torch.Generator().manual_seed(1)
    xs = [(torch.rand(4, 1, 8, 8, generator=g) > 0.5).float() for _ in range(3)]
    tr = trainer.Trainer(model=m, loss_fn=recipes.recipe_loss, optimizer=opt, train_loader=xs, eval_loader=xs[:1],
                         clip_grad_norm=0.05, skip_grad_norm=1e9, log_dir=str(tmp_path), n_gpus=1)
    return tr, opt, xs


def test_trainer_step_against_float64_and_checkpoint(tmp_path):
    tr, opt, xs = _trainer(tmp_path / "a")
    snaps = []
    step_fn = opt.clip_and_step

    def spy(max_norm, skip_above=None):
        snaps.append([(p, p.detach().clone(), p.grad.clone(),
                       opt.state[p]["ema_avg"].clone() if opt.state.get(p) else torch.zeros_like(p),
                       opt.state[p]["ema_var"].clone() if opt.state.get(p) else torch.zeros_like(p))
                      for p in tr.model.parameters()])
        return step_fn(max_norm, skip_above)

    opt.clip_and_step = spy
    for t, x in enumerate(xs, start=1):
        if t == 3:  # checkpoint after two steps; the restored trainer must take the third step bit for bit
            tr._save_checkpoint()
        metrics = tr._train_one_batch(x, None)
        assert math.isfinite(metrics["loss"])
        rows = snaps[-1]
        ref_norm, b_norm = R.sqnorm_reference([r[2] for r in rows], sum(-(-r[0].numel() // 65536) for r in rows))
        assert abs(metrics["grad_norm"] - ref_norm) <= b_norm + 1e-7 * ref_norm
        sc = R.scalars(2e-3, 0.9, 0.999, t)
        for p, p0, g0, m0, v0 in rows:
            ref = R.reference(p0, g0, m0, v0, metrics["grad_norm"], 0.05, sc)
            _within(p.detach(), ref["p"], ref["b_p"], "p")
            _within(opt.state[p]["ema_var"], ref["v"], ref["b_v"], "v")
    tr2, opt2, _ = _trainer(tmp_path / "a", seed=5)
    tr2.restore_checkpoint()
    tr2._train_one_batch(xs[2], None)
    for pa, pb in zip(tr.model.parameters(), tr2.model.parameters()):
        assert torch.equal(pa, pb)
        assert torch.equal(opt.state[pa]["ema_avg"], opt2.state[pb]["ema_avg"])
        assert opt2.state[pb]["step"] == 3


# ----------------------------------------------------------------------------------------------------------------------
# ReZero kernels
# ----------------------------------------------------------------------------------------------------------------------
def _operands(n, off, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(3):
        buf = torch.empty(n + off, device=DEV)
        buf[off:].copy_(torch.randn(n, generator=g))
        out.append(buf[off:])
    return out


@pytest.mark.parametrize("n", [1, 7, (1 << 20) + 3])
@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("alpha", [0.0, -0.75, 3e-8])
def test_rezero_kernels(fx, n, off, alpha):
    from pytorch_generative_b200 import _lib as L

    x, f, dy = _operands(n, off, n + off)
    a = torch.tensor([alpha], device=DEV)
    y = torch.empty(n + off, device=DEV)[off:]
    L.rezero_fwd(x, f, a, y)
    assert torch.equal(y, x + a * f), "forward differs from torch's x + alpha * f"
    df = torch.empty(n + off, device=DEV)[off:]
    da = torch.empty(1, device=DEV)
    n0 = L.launch_count()
    L.rezero_bwd(dy, f, a, df, da)
    assert L.launch_count() - n0 == 2
    assert torch.equal(df, dy * a)
    ref, bound = R.dalpha_bound(dy, f)
    assert abs(float(da) - ref) <= bound
    n0 = L.launch_count()
    df2 = torch.empty_like(dy)
    L.rezero_bwd(dy, f, a, df2, None)
    assert L.launch_count() - n0 == 1 and torch.equal(df2, df)


def test_rezero_bug_models_fail(fx):
    from pytorch_generative_b200 import _lib as L

    n = (1 << 20) + 3
    x, f, dy = _operands(n, 0, 1)
    a = torch.tensor([-0.75], device=DEV)
    fma = (x.double() + a.double() * f.double()).float()  # one rounding: an FMA
    assert not torch.equal(fma, x + a * f), "an FMA forward would pass the bit-for-bit test"
    ref, bound = R.dalpha_bound(dy, f)
    blocks = -(-n // L.REZERO_CHUNK)
    half = (blocks + 1) // 2 * L.REZERO_CHUNK
    partial = float((dy[:half].double() * f[:half].double()).sum())
    assert abs(partial - ref) > bound, "dalpha from the first half of the blocks would pass its bound"


# ----------------------------------------------------------------------------------------------------------------------
# ReZeroWrapper against the reference's fixture
# ----------------------------------------------------------------------------------------------------------------------
TOL = {"conv": 1e-2, "ln": 1e-3, "seq": 2e-3}  # bf16 tensor-core convolution; fp32 LayerNorm; TF32 1x1 conv


def _wrapped(fx, name):
    from pytorch_generative_b200 import nn as pnn

    module = {"conv": lambda: pnn.CausalConv2d(False, 16, 16, 3, padding=1), "ln": lambda: pnn.NCHWLayerNorm(16),
              "seq": lambda: torch.nn.Sequential(torch.nn.Conv2d(16, 16, 1), torch.nn.ReLU())}[name]()
    w = pnn.ReZeroWrapper(module)
    w.load_state_dict(fx["rezero"]["cases"][name]["state"])
    return w.to(DEV)


@pytest.mark.parametrize("name", ["conv", "ln", "seq"])
def test_rezero_wrapper_against_the_reference(fx, name):
    rz = fx["rezero"]
    case = rz["cases"][name]
    w = _wrapped(fx, name)
    x0, c = rz["x"].to(DEV), rz["c"].to(DEV)
    for alpha in (0.0, rz["alpha"]):
        with torch.no_grad():
            w._alpha.fill_(alpha)
        w.zero_grad()
        x = x0.clone().requires_grad_(True)
        y = w(x)
        (y * c).sum().backward()
        ref = case[alpha]
        if alpha == 0.0:
            assert torch.equal(y, x0) and torch.equal(x.grad, c)
            for k, p in w._module.named_parameters():
                assert torch.count_nonzero(p.grad) == 0, k
        tol = TOL[name]
        for what, got, r in [("y", y, ref["y"]), ("dx", x.grad, ref["dx"])] + \
                [(k, p.grad, ref["grads"][k]) for k, p in w._module.named_parameters()]:
            assert float((got.detach().cpu() - r).abs().max()) <= tol * max(1.0, float(r.abs().max())), (name, alpha, what)
        f_ref = (case[rz["alpha"]]["y"] - rz["x"]) / rz["alpha"]  # the module's output, the same at every alpha
        scale = float((rz["c"] * f_ref).abs().sum())
        assert abs(float(w._alpha.grad) - float(ref["dalpha"])) <= tol * max(1.0, scale), (name, alpha, "dalpha")


def test_rezero_wrapper_cuda_graph_equals_eager(fx):
    w = _wrapped(fx, "conv")
    params = [w._alpha] + list(w._module.parameters())
    x = fx["rezero"]["x"].to(DEV).requires_grad_(True)
    c = fx["rezero"]["c"].to(DEV)

    def step():
        y = w(x)
        return (y.detach(),) + torch.autograd.grad((y * c).sum(), [x] + params)

    with torch.no_grad():
        w._alpha.fill_(0.5)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for alpha in (0.5, -1.25, 0.0, 3e-3):
        with torch.no_grad():
            w._alpha.fill_(alpha)
        graph.replay()
        eager = step()
        for a, b in zip(outs, eager):
            assert torch.equal(a, b), alpha
