"""VQ-VAE, VQ-VAE-2 and VectorQuantizer on the H100: the quantizer kernels, the code sums, the EMA update, the
backward and the MSE against float64 with per-element bounds; both models against the reference's outputs, indices
and buffers (tests/golden/vq_vae.pt) and every gradient against a float64 restatement that takes the device's bf16
roundings and indices; eval() without updates, determinism, pad columns, a FusedAdam trajectory, the step under a CUDA
graph, both recipes, and deepcopy / pickle after a step."""

import copy
import os
import pickle

import pytest
import torch

import _vq_vae_reference as R
from _conv_stack_reference import assign_bound

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vq_vae.pt")
TOL = 1e-2
U32 = 2.0 ** -24
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
# Per tensor, relative to its own largest entry.  Measured on an H100: at most 0.74% on the fixtures and 5.0% at the
# recipe size (VQ-VAE-2's encoder_t residual block).  A zero gradient is off by 100%, a wrong sign by 200%.
GRAD_TOL, FIXTURE_GRAD_TOL = 0.25, 0.05


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture
def recorded_idx(monkeypatch):
    """Records the indices of every pg_vq_assign call, in call order."""
    from pytorch_generative_b200 import _lib as L

    calls = []
    orig = L.vq_assign

    def rec(x, emb, idx, *args, **kwargs):
        orig(x, emb, idx, *args, **kwargs)
        calls.append(idx)
    monkeypatch.setattr(L, "vq_assign", rec)
    return calls


def _err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _within(got, ref, bound, what):
    d = (got.double().cpu() - ref.double().cpu()).abs()
    bad = d > bound.double().cpu()
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} entries out of bounds, worst excess {(d - bound.cpu()).max().item():.3e}"


# --------------------------------------------------------------------------------------------------
# kernels
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 7, 512, 1000])
@pytest.mark.parametrize("d", [1, 6, 64, 100])
def test_assign_against_float64(K, d):
    """The chosen code's float64 distance is within the fp32 rounding bound of the float64 optimum; the operand at a
    column offset and pitch, its zero pad and the commitment sum are held per element.  1000 codes of 64 or 100
    columns exceed one shared-memory chunk; 100 columns take the path without a register row."""
    from pytorch_generative_b200 import _lib as L

    torch.manual_seed(K * 131 + d)
    P = 333  # not a multiple of the 64-row tile
    x = torch.randn(P, d + 3, device=dev())[:, :d]  # a pitch wider than the row
    emb = torch.randn(K, d, device=dev())
    idx = torch.empty(P, dtype=torch.int32, device=dev())
    col0, out_cols, ld = 5, d + 4, d + 16
    out = torch.full((P, ld), float("nan"), dtype=BF16, device=dev())
    acc = torch.zeros(1, device=dev())
    L.vq_assign(x, emb, idx, out, col0, out_cols, acc)
    xd, ed = x.double(), emb.double()
    dist = (xd * xd).sum(1, keepdim=True) + (ed * ed).sum(1) - 2 * xd @ ed.t()
    bound = assign_bound(xd, ed)  # per code, twice for the comparison of two codes
    chosen = idx.long()
    best = dist.min(1).values
    got = dist.gather(1, chosen[:, None])[:, 0]
    assert bool((chosen >= 0).all() and (chosen < K).all())
    _within(got, best, bound.gather(1, chosen[:, None])[:, 0] + bound.max(1).values, "chosen distance")
    q = ed[chosen]
    st = (xd.float() + (q.float() - xd.float())).double()
    assert torch.equal(out[:, col0:col0 + d].double(), st.to(BF16).double()), "operand"
    assert not bool(out[:, col0 + d:col0 + out_cols].float().any()), "pad columns"
    assert bool(out[:, :col0].isnan().all() and out[:, col0 + out_cols:].isnan().all()), "columns outside the window"
    ref = ((xd - q) ** 2).sum()
    _within(acc, ref.view(1), (P * d + 2) * U32 * ref.view(1) + 1e-30, "commitment sum")


def test_assign_ties_keep_the_lowest_index():
    """Integer inputs make every distance exact: duplicated codes tie exactly and the lowest index wins, as
    torch.argmin's first minimum."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(3)
    for K, d in ((7, 6), (512, 64), (1000, 9)):
        base = torch.randint(-3, 4, (K // 2 + 1, d), generator=g).float()
        emb = torch.cat([base, base])[:K]  # every code of the first half appears twice
        emb = emb[torch.randperm(K, generator=g)].contiguous().to(dev())
        x = torch.randint(-3, 4, (517, d), generator=g).float().to(dev())
        idx = torch.empty(517, dtype=torch.int32, device=dev())
        L.vq_assign(x, emb, idx)
        xd, ed = x.double(), emb.double()
        dist = (xd * xd).sum(1, keepdim=True) + (ed * ed).sum(1) - 2 * xd @ ed.t()
        assert torch.equal(idx.long(), dist.argmin(1)), (K, d)
        assert int((dist == dist.min(1, keepdim=True).values).sum(1).max()) >= 2, "the test has ties"


@pytest.mark.parametrize("K, d, P", [(512, 64, 8192), (10, 6, 37), (7, 130, 200), (1, 1, 5)])
def test_code_sums_ema_and_codebook_gradient_against_float64(K, d, P):
    """Given the device's indices: counts exact, sums within the fp32 bound of an ordered sum, the EMA update and the
    use_ema=False codebook gradient per element, codes with no rows included."""
    from pytorch_generative_b200 import _lib as L

    torch.manual_seed(K + d + P)
    x = torch.randn(P, d, device=dev())
    emb = torch.randn(K, d, device=dev())
    idx = torch.randint(0, max(1, K // 2), (P,), dtype=torch.int32, device=dev())  # half the codes get no row
    counts = torch.full((K,), float("nan"), device=dev())
    sums = torch.full((K, d), float("nan"), device=dev())
    L.vq_code_sums(x, idx, K, sums, counts)
    one_hot = torch.zeros(P, K, dtype=F64, device=dev())
    one_hot[torch.arange(P), idx.long()] = 1
    assert torch.equal(counts.double(), one_hot.sum(0))
    want = one_hot.t() @ x.double()
    sabs = one_hot.t() @ x.double().abs()
    _within(sums, want, P * U32 * sabs + 1e-30, "sums")
    cs, avg, e = torch.rand(K, device=dev()), torch.randn(K, d, device=dev()), emb.clone()
    cs0, avg0 = cs.double(), avg.double()
    L.vq_ema_update(counts, sums, 0.99, cs, avg, e)
    cs_ref = cs0 * 0.99 + counts.double() * (1 - 0.99)
    avg_ref = avg0 * 0.99 + sums.double() * (1 - 0.99)
    _within(cs, cs_ref, 4 * U32 * cs_ref.abs(), "cluster size")
    _within(avg, avg_ref, 4 * U32 * (avg0.abs() + sums.double().abs()), "embedding avg")
    e_ref = avg.double() / (cs.double() + 1e-5)[:, None]
    _within(e, e_ref, 4 * U32 * e_ref.abs(), "embedding")
    g = torch.tensor([0.7], device=dev())
    grad = torch.full((K, d), float("nan"), device=dev())
    L.vq_code_sums(x, idx, K, grad, emb=emb, g=g, scale=2.0 / (P * d))
    v = (emb.double()[idx.long()] - x.double()) * (2.0 / (P * d)) * 0.7
    want = one_hot.t() @ v
    _within(grad, want, (P + 4) * U32 * (one_hot.t() @ v.abs()) + 1e-30, "codebook gradient")
    assert not bool(grad[K // 2 + 1:].any()) and not bool(sums[max(1, K // 2):].any())


@pytest.mark.parametrize("dtype", [BF16, F32])
def test_vq_bwd_and_mse_against_float64(dtype):
    from pytorch_generative_b200 import _lib as L

    torch.manual_seed(9)
    P, d, K = 301, 6, 10
    x = torch.randn(P, d, device=dev())
    emb = torch.randn(K, d, device=dev())
    idx = torch.randint(0, K, (P,), dtype=torch.int32, device=dev())
    dq = torch.randn(P, 16, device=dev()).to(dtype)
    g = torch.tensor([1.3], device=dev())
    ld = 8 if dtype == BF16 else d
    dx = torch.full((P, ld), float("nan"), dtype=dtype, device=dev())
    L.vq_bwd(x, emb, idx, dq, 6, g, 2.0 / (P * d), dx)
    commit = (x.double() - emb.double()[idx.long()]) * (2.0 / (P * d)) * 1.3
    want = dq[:, 6:12].double() + commit
    u = 2.0 ** -8 if dtype == BF16 else U32
    _within(dx[:, :d], want, u * want.abs() + 4 * U32 * (commit.abs() + dq[:, 6:12].double().abs()), "dx")
    assert not bool(dx[:, d:].float().any()), "dx pad columns"
    # mse: two pitches, the pad columns of the gradients zero
    a = torch.randn(1000, 16, device=dev())
    b = torch.randn(1000, 12, device=dev())
    acc = torch.zeros(1, device=dev())
    L.mse_mean(a, b, 12, loss_sum=acc)
    diff = a[:, :12].double() - b.double()
    _within(acc, (diff ** 2).sum().view(1), 12000 * U32 * (diff ** 2).sum().view(1), "mse sum")
    da = torch.full_like(a, float("nan"))
    db = torch.full_like(b, float("nan"))
    L.mse_mean(a, b, 12, g=g, scale=2.0 / 12000, da=da, db=db)
    want = diff * (2.0 / 12000) * 1.3
    _within(da[:, :12], want, 4 * U32 * want.abs(), "da")
    assert torch.equal(db, -da[:, :12]) and not bool(da[:, 12:].any())


def test_standalone_quantizer_without_ema(fixture):
    """nn.VectorQuantizer(use_ema=False) on NCHW: outputs, loss, the input and codebook gradients against the
    reference at 1e-2 (fp32 throughout: no bf16 operand on this path)."""
    from pytorch_generative_b200 import nn

    fx = fixture["vq_no_ema"]
    m = nn.VectorQuantizer(**fx["kwargs"]).to(dev())
    m.load_state_dict(fx["state"])
    x = fx["x"].to(dev()).requires_grad_(True)
    q, loss = m(x)
    ((q * fx["cot"].to(dev())).sum() + loss).backward()
    assert _err(q, fx["outputs"]) <= 1e-5 and _err(loss, fx["vq_loss"]) <= 1e-5
    assert _err(x.grad, fx["x_grad"]) <= 1e-5 and _err(m._embedding.grad, fx["grads"]["_embedding"]) <= 1e-5


# --------------------------------------------------------------------------------------------------
# the models
# --------------------------------------------------------------------------------------------------
def _loaded(fx):
    from pytorch_generative_b200 import models

    m = getattr(models, fx["cls"])(**fx["kwargs"])
    m.load_state_dict(fx["state"])
    return m.to(dev()).train(fx["train"])


def _names(fx):
    """The quantizers in the order the CUDA path calls them."""
    return ["_quantizer_t._net.1", "_quantizer_b._net.1"] if fx["cls"] == "VectorQuantizedVAE2" else ["_quantizer._net.1"]


def _loss(fx, out):
    from pytorch_generative_b200 import losses

    return (losses.vq_vae_loss if fx["cls"] == "VectorQuantizedVAE" else losses.vq_vae_2_loss)(out[2], None, out[:2])


def _grads_close(got, ref, what, tol):
    ratios = []
    for k, r in ref.items():
        g, r = got[k].detach().double().cpu(), r.detach().double().cpu()
        ratios.append(((g - r).abs().max().item() / max(r.abs().max().item(), 1e-30), k))
    ratios.sort(reverse=True)
    assert ratios[0][0] <= tol, (what, ratios[:5])
    return ratios


@pytest.mark.parametrize("name", ["vq_vae", "vq_vae_eval", "vq_vae_2"])
def test_the_reference_outputs(fixture, recorded_idx, name):
    """Outputs, vq_loss, the loss dict and the buffers after the forward against the reference at 1e-2, with the
    reference's indices; every gradient against the float64 restatement given the device's bf16 roundings and indices,
    each tensor within FIXTURE_GRAD_TOL of its own largest entry."""
    fx = fixture[name]
    m = _loaded(fx)
    x = fx["x"].to(dev())
    x_hat, vq_loss = m(x)
    out = _loss(fx, (x_hat, vq_loss, x))
    out["loss"].backward()
    names = _names(fx)
    assert len(recorded_idx) == len(names)
    idx = dict(zip(names, (i.long().cpu() for i in recorded_idx)))
    for k in names:
        assert torch.equal(idx[k], fx["vq_inputs"][k]["idx"]), (name, k)
    assert _err(x_hat, fx["outputs"]) <= TOL and _err(vq_loss, fx["vq_loss"]) <= TOL, name
    for k, v in fx["losses"].items():
        assert _err(out[k], v) <= TOL, (name, k)
    sd = m.state_dict()
    for k, v in fx["buffers"].items():
        assert _err(sd[k], v) <= TOL, (name, k)
    _, _, ref, _ = R.run(fx, F64, dev(), R.device_rounding, idx)
    ratios = _grads_close({k: p.grad for k, p in m.named_parameters()}, ref, name, FIXTURE_GRAD_TOL)
    print(name, "worst gradient errors over own scale:", ratios[:3])


@pytest.mark.parametrize("cls, residual", [("VectorQuantizedVAE", 32), ("VectorQuantizedVAE2", 64)])
def test_recipe_size_against_the_restatement(recorded_idx, cls, residual):
    """The recipe's widths at batch 2 on 3x32x32: outputs and loss against the fp32 restatement (given the device's
    indices) at 1e-2, every gradient against the float64 restatement with the device's roundings and indices, each
    tensor within GRAD_TOL of its own largest entry."""
    from pytorch_generative_b200 import models

    torch.manual_seed(5)
    kw = dict(in_channels=3, out_channels=3, hidden_channels=128, n_residual_blocks=2, residual_channels=residual,
              n_embeddings=512, embedding_dim=64)
    m = getattr(models, cls)(**kw).to(dev())
    state = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(6)).to(dev())
    fx = dict(cls=cls, kwargs=kw, train=True, x=x, state=state)
    x_hat, vq_loss = m(x)
    out = _loss(fx, (x_hat, vq_loss, x))
    out["loss"].backward()
    idx = dict(zip(_names(fx), (i.long() for i in recorded_idx)))
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        r_out, r_losses, _, _ = R.run(fx, F32, dev(), idx=idx)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    assert _err(x_hat, r_out) <= TOL
    for k in ("vq_loss", "reconstruction_loss", "loss"):
        assert _err(out[k], r_losses[k]) <= TOL, k
    _, _, ref, _ = R.run(fx, F64, dev(), R.device_rounding, idx)
    ratios = _grads_close({k: p.grad for k, p in m.named_parameters()}, ref, cls, GRAD_TOL)
    print(cls, "worst gradient errors over own scale:", ratios[:5])


def test_eval_leaves_the_buffers_and_launches_no_update(fixture):
    from pytorch_generative_b200 import _lib as L

    fx = fixture["vq_vae_2"]
    m = _loaded(fx)
    x = fx["x"].to(dev())
    m._register_shape(*x.shape[1:])
    m.eval()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    with torch.no_grad():
        m(x)  # builds the bf16 weight copies, which later forwards reuse
    n0 = L.launch_count()
    with torch.no_grad():
        m(x)
    n_eval = L.launch_count() - n0
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k
    m.train()
    n0 = L.launch_count()
    with torch.no_grad():
        m(x)
    assert L.launch_count() - n0 == n_eval + 2 * 2, "train adds pg_vq_code_sums and pg_vq_ema_update per quantizer"
    assert not torch.equal(m.state_dict()["_quantizer_b._net.1._cluster_size"], before["_quantizer_b._net.1._cluster_size"])


@pytest.mark.parametrize("name", ["vq_vae", "vq_vae_2"])
def test_repeat_runs_are_bit_identical(fixture, name):
    fx = fixture[name]
    runs = []
    for _ in range(2):
        m = _loaded(fx)
        x_hat, vq_loss = m(fx["x"].to(dev()))
        (x_hat.sum() + vq_loss).backward()
        runs.append([x_hat.detach(), vq_loss.detach()] + [p.grad for p in m.parameters()] + list(m.buffers()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_pad_columns_are_exactly_zero(fixture):
    """VQ-VAE-2's decoder_b operand cat(_conv(decoded_t), quantized_b) of 2 x 5 columns in a 16-column pitch: zero in
    columns 10..15; the quantizer keeps _conv's columns; the gradient of z leaves in bf16."""
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.nn import pm

    fx = fixture["vq_vae_2"]
    m = _loaded(fx)
    P = 16
    left = torch.randn(P, 5, device=dev()).to(BF16)
    z = torch.randn(P, 16, device=dev()).requires_grad_(True)
    cat, loss = m._quantizer_b._pm(z, pm.Geom(1, 4, 4), left=left)
    assert cat.shape == (P, 16) and torch.equal(cat[:, :5], left) and not bool(cat[:, 10:].float().any())
    seen = []
    conv, vq = m._quantizer_b._net
    zz, zb = pm.conv(z, conv.weight, conv.bias, pm.Geom(1, 4, 4), out_f32=True, emit=L.ACT_NONE, emit_mode=pm.POST)
    zb.register_hook(lambda g: seen.append(g.dtype))
    out, loss = vq._pm(zb, zz.detach(), 8)
    assert out.shape == (P, 8) and not bool(out[:, 5:].float().any())
    (out.float().sum() + loss).backward()
    assert seen == [BF16]


def test_fused_adam_trajectory_matches_the_restatement(fixture, recorded_idx):
    """Three FusedAdam steps against torch.optim.Adam on the float64 restatement given the device's roundings and
    indices: losses, each parameter's update within ADAM_TOL of its own norm, and the EMA buffers at 1e-2."""
    from pytorch_generative_b200 import optim

    ADAM_TOL = 0.25
    fx = dict(fixture["vq_vae_2"])
    m = _loaded(fx)
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    state = {k: v.to(dev(), F64) for k, v in fx["state"].items()}
    params = {k: v.clone().requires_grad_(True) for k, v in state.items() if R.is_param(k)}
    ref_opt = torch.optim.Adam(list(params.values()), lr=2e-4)
    opt = optim.FusedAdam(m.parameters(), lr=2e-4)
    for s in range(3):
        x = torch.randn(1, 3, 8, 8, generator=torch.Generator().manual_seed(40 + s)).to(dev())
        recorded_idx.clear()
        opt.zero_grad()
        out = _loss(fx, (*m(x), x))
        out["loss"].backward()
        opt.clip_and_step(1e50)
        idx = dict(zip(_names(fx), (i.long() for i in recorded_idx)))
        ref_opt.zero_grad()
        cur = {**state, **params}
        x_hat, vq_loss, found = R.vq_vae_2(cur, x.double(), R.device_rounding, True, idx)
        ref_loss = R.loss_fn(x.double(), x_hat, vq_loss, 0.25)["loss"]
        ref_loss.backward()
        ref_opt.step()
        for k, f in found.items():
            for b, n in zip(f["buffers"], ("_cluster_size", "_embedding_avg", "_embedding")):
                state[f"{k}.{n}"] = b.detach()
        assert abs(out["loss"].item() - ref_loss.item()) <= TOL * max(1.0, abs(ref_loss.item())), s
    sd = m.state_dict()
    for k, v in state.items():
        if not R.is_param(k):
            assert _err(sd[k], v) <= TOL, k
    ratios = sorted((((p.detach() - before[k]).double() - (params[k].detach() - fx["state"][k].to(dev(), F64))).norm().item()
                     / (params[k].detach() - fx["state"][k].to(dev(), F64)).norm().item(), k) for k, p in m.named_parameters())
    print("worst update errors over own norm:", ratios[-5:])
    assert ratios[-1][0] <= ADAM_TOL, ratios[-5:]


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

    return losses.vq_vae_2_loss(x, None, preds)["loss"]


def test_graphed_train_step_equals_the_eager_step():
    """The step, the EMA updates included, never synchronises with the host: three replays equal three eager steps bit
    for bit, parameters and buffers."""
    from pytorch_generative_b200 import models, trainstep

    torch.manual_seed(7)
    init = models.VectorQuantizedVAE2(3, 3, 32, 1, 16, 64, 8).to(dev())
    state = {k: v.clone() for k, v in init.state_dict().items()}
    g = torch.Generator().manual_seed(8)
    xs = [torch.randn(8, 3, 16, 16, generator=g).to(dev()) for _ in range(3)]
    graphed = _TupleModel(copy.deepcopy(init))
    step = trainstep.GraphedTrainStep(graphed, graphed.parameters(), _tuple_loss, xs[0], lr=2e-4, lr_gamma=1.0)
    step.reset({f"model.{k}": v for k, v in state.items()}, lr=2e-4)
    eager = _TupleModel(copy.deepcopy(init))
    eager.model.load_state_dict(state)
    params = list(eager.parameters())
    opt = torch.optim.Adam(params, lr=torch.tensor(2e-4, device=dev()), capturable=True)
    for x in xs:
        loss_g, norm_g = step(x)
        opt.zero_grad(set_to_none=True)
        loss = _tuple_loss(eager(x), x)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(params, 1e50, foreach=True)
        opt.step()
        assert loss_g == loss.item() and norm_g == norm.item()
    for (k, a), b in zip(graphed.state_dict().items(), eager.state_dict().values()):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("name, cls", [("vq_vae", "VectorQuantizedVAE"), ("vq_vae_2", "VectorQuantizedVAE2")])
def test_recipe_trains_one_epoch_and_checkpoints(tmp_path, name, cls):
    from pytorch_generative_b200 import models, recipes

    g = torch.Generator().manual_seed(50)
    loader = [(torch.randn(8, 3, 32, 32, generator=g).to(dev()), None) for _ in range(2)]
    trainer = getattr(recipes, f"reproduce_{name}")(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["optimizer"]["param_groups"][0]["lr"] == pytest.approx(2e-4 * 0.999977 ** 1, rel=1e-9) or \
        ckpt["optimizer"]["param_groups"][0]["initial_lr"] == 2e-4
    fresh = getattr(models, cls)(3, 3, 128, 2, 32 if name == "vq_vae" else 64, 512, 64)
    fresh._register_shape(3, 32, 32)
    assert sorted(ckpt["model"]) == sorted(fresh.state_dict())
    live = trainer.model.state_dict()
    for k, v in ckpt["model"].items():
        if k.endswith("_cluster_size"):
            assert bool(v.any()) and torch.equal(v.to(dev()), live[k]), k


def test_deepcopy_and_pickle_after_a_step(fixture):
    from pytorch_generative_b200 import optim

    fx = fixture["vq_vae"]
    m = _loaded(fx)
    opt = optim.FusedAdam(m.parameters(), lr=2e-4)
    x = fx["x"].to(dev())
    x_hat, vq_loss = m(x)
    (x_hat.square().mean() + vq_loss).backward()
    opt.clip_and_step(1e50)
    for clone in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        for k, v in m.state_dict().items():
            assert torch.equal(clone.state_dict()[k], v), k
        with torch.no_grad():
            assert torch.equal(clone.eval()(x)[0], m.eval()(x)[0])
        m.train()
