"""CPU checks of AdaBelief and ReZeroWrapper: the float64 restatement against the reference's trajectory (and its bug
models against it), the optimizer's constructor, param groups and state-dict layout, ReZeroWrapper's state dict,
shape and device checks, and the overlay bindings."""

import os
import sys

import pytest
import torch

import _adabelief_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "adabelief_rezero.pt")


@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLD, weights_only=False)


def _trajectory_errors(fx, bug=None):
    """Largest |restatement - fixture| / max|restatement| over every step, stepped parameter and p / m / v."""
    ab = fx["adabelief"]
    init = R.initial_params()
    worst = 0.0
    for t, rec in enumerate(ab["steps"], start=1):
        grads = R.grads_at(t)
        prev = None if t == 1 else ab["steps"][t - 2]
        for k in rec["p"]:
            p0 = init[k] if prev is None else R.unpack(prev["p"][k])
            m0 = torch.zeros_like(p0) if prev is None else R.unpack(prev["m"][k])
            v0 = torch.zeros_like(p0) if prev is None else R.unpack(prev["v"][k])
            gr = R.group_of(k)
            sc = R.scalars(gr["lr"], *gr["betas"], rec["step"][k])
            out = R.reference(p0, grads[k], m0, v0, rec["norm"], rec["max_norm"], sc, bug=bug)
            for key in ("p", "m", "v"):
                ref = out[key]
                scale = float(ref.abs().max()) or 1e-30
                worst = max(worst, float((ref - R.unpack(rec[key][k]).double()).abs().max()) / scale)
    return worst


def test_restatement_follows_the_reference_trajectory(fx):
    assert all(rec["step"]["a"] == t for t, rec in enumerate(fx["adabelief"]["steps"], start=1))
    assert _trajectory_errors(fx) <= 1e-6


@pytest.mark.parametrize("bug", R.BUGS)
def test_bug_models_miss_the_reference_trajectory(fx, bug):
    assert _trajectory_errors(fx, bug) > 100 * 1e-6


def test_fixture_inputs_rebuild():
    assert R.grads_at(1)["none"] is None
    big = R.initial_params()["big"]
    assert big.numel() == 70000 and torch.equal(big[R.PERIOD:2 * R.PERIOD], big[:R.PERIOD])
    d = R.pack(big)
    assert d["idx"].numel() == 0 and torch.equal(R.unpack(d), big)
    bumped = big.clone()
    bumped[69999] += 1
    assert torch.equal(R.unpack(R.pack(bumped)), bumped)
    assert set(R.SIZES) == {n for gr in R.GROUPS for n in gr["names"]}


def test_constructor_checks_and_param_groups():
    from pytorch_generative_b200.optim import AdaBelief

    p = [torch.nn.Parameter(torch.zeros(3))]
    for kwargs in (dict(lr=-1e-3), dict(betas=(1.0, 0.9)), dict(betas=(-0.1, 0.9)), dict(betas=(0.9, 1.0))):
        with pytest.raises(AssertionError):
            AdaBelief(p, **kwargs)
    opt = AdaBelief(p)
    assert len(opt.param_groups) == 1
    assert set(opt.param_groups[0]) == {"lr", "betas", "params"}
    assert opt.param_groups[0]["lr"] == 1e-3 and opt.param_groups[0]["betas"] == (0.9, 0.999)


def _params():
    return {k: torch.nn.Parameter(v.clone()) for k, v in R.initial_params().items()}


def _groups(params):
    return [dict(params=[params[n] for n in gr["names"]], lr=gr["lr"], betas=gr["betas"]) for gr in R.GROUPS]


def test_reference_state_dicts_load_and_keep_their_layout(fx):
    from pytorch_generative_b200.optim import AdaBelief

    for key in (0, 3):
        ref_sd = R.unpack_state_dict(fx["adabelief"]["state_dicts"][key])
        opt = AdaBelief(_groups(_params()))
        opt.load_state_dict(ref_sd)
        sd = opt.state_dict()
        assert [set(g) for g in sd["param_groups"]] == [set(g) for g in ref_sd["param_groups"]]
        assert [g["params"] for g in sd["param_groups"]] == [g["params"] for g in ref_sd["param_groups"]]
        assert sorted(sd["state"]) == sorted(ref_sd["state"])
        for i, st in sd["state"].items():
            ref_st = ref_sd["state"][i]
            assert list(st) == list(ref_st) == ["step", "ema_avg", "ema_var"]
            assert type(st["step"]) is int and st["step"] == ref_st["step"] == key
            for n in ("ema_avg", "ema_var"):
                assert st[n].dtype == torch.float32 and torch.equal(st[n], ref_st[n])
    # the parameter without gradient never got state
    assert len(fx["adabelief"]["state_dicts"][3]["state"]) == len(R.SIZES) - 1


def _our_module(name):
    from pytorch_generative_b200 import nn as pnn

    if name == "conv":
        return pnn.CausalConv2d(False, 16, 16, 3, padding=1)
    if name == "ln":
        return pnn.NCHWLayerNorm(16)
    return torch.nn.Sequential(torch.nn.Conv2d(16, 16, 1), torch.nn.ReLU())


@pytest.mark.parametrize("name", ["conv", "ln", "seq"])
def test_rezero_state_dict_matches_the_reference(fx, name):
    from pytorch_generative_b200.nn import ReZeroWrapper

    case = fx["rezero"]["cases"][name]
    w = ReZeroWrapper(_our_module(name))
    sd = w.state_dict()
    assert list(sd) == case["keys"]
    assert {k: tuple(v.shape) for k, v in sd.items()} == case["shapes"]
    assert w._alpha.dtype == torch.float32 and torch.equal(w._alpha.detach(), case["alpha0"])
    assert w._alpha.detach().view(torch.int32).item() == 0  # +0.0, bit for bit
    w.load_state_dict(case["state"])  # a reference checkpoint loads as is
    assert [n for n, _ in w.named_parameters()][0] == "_alpha"


def test_rezero_refuses_a_shape_change_and_cpu_tensors():
    from pytorch_generative_b200.nn import ReZeroWrapper

    w = ReZeroWrapper(torch.nn.Conv2d(4, 8, 1))
    with pytest.raises(ValueError, match=r"\(1, 8, 3, 3\).*\(1, 4, 3, 3\)"):
        w(torch.zeros(1, 4, 3, 3))
    with pytest.raises(RuntimeError):
        ReZeroWrapper(torch.nn.Identity())(torch.zeros(1, 4, 3, 3))


def test_adabelief_refuses_cpu_and_sparse():
    from pytorch_generative_b200.optim import AdaBelief

    p = torch.nn.Parameter(torch.zeros(3))
    p.grad = torch.ones(3)
    with pytest.raises(RuntimeError, match="CUDA"):
        AdaBelief([p]).step()
    p.grad = torch.ones(3).to_sparse()
    with pytest.raises(RuntimeError, match="sparse"):
        AdaBelief([p]).step()


def _stand_in(root, with_names):
    """A minimal reference package: the names overlay.install() always binds, plus optim.AdaBelief and
    nn.utils.ReZeroWrapper (exported from nn) when `with_names`."""
    pkg = root / "pytorch_generative"
    (pkg / "models" / "autoregressive").mkdir(parents=True)
    (pkg / "nn").mkdir()
    (pkg / "__init__.py").write_text("from pytorch_generative import models, nn\n")
    nn_names = ["CausalConv2d", "GatedActivation", "NCHWLayerNorm", "CausalAttention", "LinearCausalAttention"]
    nn_init = "".join(f"class {n}:\n    pass\n" for n in nn_names) + "def image_positional_encoding(shape):\n    pass\n"
    if with_names:
        (pkg / "nn" / "utils.py").write_text("class ReZeroWrapper:\n    pass\n")
        nn_init += "from pytorch_generative.nn.utils import ReZeroWrapper\n"
        (pkg / "optim.py").write_text("class AdaBelief:\n    pass\n")
    (pkg / "nn" / "__init__.py").write_text(nn_init)
    mods = {"pixel_cnn": "PixelCNN", "gated_pixel_cnn": "GatedPixelCNN", "pixel_snail": "PixelSNAIL", "image_gpt": "ImageGPT"}
    for mod, cls in mods.items():
        (pkg / "models" / "autoregressive" / f"{mod}.py").write_text(f"class {cls}:\n    pass\n")
    (pkg / "models" / "autoregressive" / "__init__.py").write_text("")
    (pkg / "models" / "__init__.py").write_text(
        "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items()))


@pytest.mark.parametrize("with_names", [True, False])
def test_overlay_binds_adabelief_and_rezero_where_the_reference_has_them(tmp_path, with_names):
    _stand_in(tmp_path, with_names)
    sys.path.insert(0, str(tmp_path))
    try:
        import importlib

        import pytorch_generative as ref

        from pytorch_generative_b200 import nn, optim, overlay

        bound = overlay.install()
        try:
            extra = {"pytorch_generative.optim.AdaBelief", "pytorch_generative.nn.ReZeroWrapper",
                     "pytorch_generative.nn.utils.ReZeroWrapper"}
            assert len(bound) == 14 + (3 if with_names else 0)
            assert extra & set(bound) == (extra if with_names else set())
            if with_names:
                assert importlib.import_module("pytorch_generative.optim").AdaBelief is optim.AdaBelief
                assert ref.nn.ReZeroWrapper is nn.ReZeroWrapper
                assert importlib.import_module("pytorch_generative.nn.utils").ReZeroWrapper is nn.ReZeroWrapper
        finally:
            overlay.uninstall()
        if with_names:
            assert importlib.import_module("pytorch_generative.optim").AdaBelief is not optim.AdaBelief
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
