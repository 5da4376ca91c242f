"""GaussianProcess without a GPU: the restatement (tests/_gp_reference.py) against the reference's own outputs
(tests/golden/gp.pt), the float64 semi-definite Cholesky, the constructor, the noise_var buffer, state-dict keys, fit,
the prior, the refusals, the overlay binding, pickle / deepcopy and the C ABI."""

import copy
import os
import pickle
import sys

import pytest
import torch

import _gp_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "gp.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def test_fixture_is_small():
    assert os.path.getsize(GOLD) < 1 << 20


def test_restatement_matches_the_reference_bit_for_bit(fixture):
    for name, case in fixture.items():
        steps, mu, sig, grads = R.replay(case, R.reference_predict)
        assert len(steps) == len(case["steps"]), name
        for (m, s), (fm, fs) in zip(steps, case["steps"]):
            assert torch.equal(m, fm) and torch.equal(s, fs), name
        assert list(grads) == list(case["grads"]) == ["x", "train_x", "train_y", "c", "s", "ell"]
        for k, g in case["grads"].items():
            assert grads[k].dtype == g.dtype and torch.equal(grads[k], g), (name, k)


def test_psd_cholesky_agrees_with_the_reference_posterior(fixture):
    """The float64 Cholesky posterior equals the reference's LU posterior to rounding on the fp64 cases."""
    for name in ("notebook", "d3", "multi"):
        case = fixture[name]
        p = case["params"]
        mean, kernel = R.ConstMean(p["c"]), R.SqExp(p["s"], p["ell"])
        tx = torch.cat([f[0] for f in case["fits"]])
        ty = torch.cat([f[1] for f in case["fits"]])
        x = case["x"]
        with torch.no_grad():
            mu, sig = R.cholesky_predict(kernel(tx, tx), kernel(tx, x), kernel(x, x), ty - mean(tx), mean(x),
                                         float(torch.tensor(case["noise"])))
        fm, fs = case["steps"][-1]
        assert torch.allclose(mu, fm, rtol=0, atol=1e-8 * fm.abs().max()), name
        assert torch.allclose(sig, fs, rtol=0, atol=1e-8 * fs.abs().max()), name


def test_psd_cholesky_drops_dependent_pivots():
    x = torch.linspace(0, 6, 100, dtype=torch.float64)[:, None]
    K = R.SqExp()(x, x).detach()
    L, dropped = R.psd_cholesky(K)
    assert dropped > 0 and torch.isfinite(L).all()
    dup = torch.cat([x[:5], x[2:3]])
    L, dropped = R.psd_cholesky(R.SqExp()(dup, dup).detach())
    assert dropped == 1 and torch.all(L[:, 5] == 0)


def test_constructor_buffer_and_state_dict():
    from pytorch_generative_b200.models import GaussianProcess

    gp = GaussianProcess(R.ConstMean(), R.SqExp())
    assert gp.noise_var.dtype == torch.float32 and float(gp.noise_var) == 0.0
    assert list(gp.state_dict()) == ["noise_var", "mean.c", "kernel.s", "kernel.ell"]
    assert gp.train_x is None and gp.train_y is None
    gp = GaussianProcess(lambda x: x, lambda a, b: a @ b.T, 0.1 ** 2)
    assert gp.noise_var.dtype == torch.float32 and gp.noise_var.item() == torch.tensor(0.01).item()
    assert list(gp.state_dict()) == ["noise_var"]
    assert GaussianProcess(R.ConstMean(), R.SqExp(), 0.5).double().noise_var.dtype == torch.float64


def test_fit_concatenates_and_the_prior_is_the_callables_output():
    from pytorch_generative_b200.models import GaussianProcess

    mean, kernel = R.ConstMean(0.5), R.SqExp()
    gp = GaussianProcess(mean, kernel)
    x = torch.rand(7, 2)
    mu, sig = gp.predict(x)
    assert torch.equal(mu, mean(x)) and torch.equal(sig, kernel(x, x))
    sentinel = object()
    gp2 = GaussianProcess(lambda x: sentinel, lambda a, b: (a, b))
    assert gp2.predict(x)[0] is sentinel and gp2.predict(x)[1][0] is x
    a, b = torch.rand(3, 2), torch.rand(2, 2)
    gp.fit(a, torch.rand(3, 1))
    assert gp.train_x is a
    gp.fit(b, torch.rand(2, 1))
    assert torch.equal(gp.train_x, torch.cat([a, b])) and gp.train_y.shape == (5, 1)


def test_cpu_and_integer_refusals_after_fit():
    from pytorch_generative_b200.models import GaussianProcess

    gp = GaussianProcess(R.ConstMean(), R.SqExp(), 0.01)
    gp.fit(torch.rand(4, 2), torch.rand(4, 1))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gp.predict(torch.rand(3, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gp.sample(torch.rand(3, 2), 2)
    gi = GaussianProcess(lambda x: torch.zeros(x.shape[0], 1, dtype=torch.int64),
                         lambda a, b: torch.ones(a.shape[0], b.shape[0], dtype=torch.int64))
    gi.fit(torch.zeros(4, 2, dtype=torch.int64), torch.zeros(4, 1, dtype=torch.int64))
    with pytest.raises(RuntimeError):
        gi.predict(torch.zeros(3, 2, dtype=torch.int64))


def test_sample_refuses_several_outputs_before_any_kernel():
    from pytorch_generative_b200.models import GaussianProcess

    gp = GaussianProcess(lambda x: torch.zeros(x.shape[0], 3), R.SqExp())
    with pytest.raises(ValueError):
        gp.sample(torch.rand(5, 2), 4)


def test_pickle_and_deepcopy_keep_the_training_data():
    from pytorch_generative_b200.models import GaussianProcess

    gp = GaussianProcess(R.ConstMean(0.3), R.SqExp(1.2, 0.4), 0.02)
    gp.fit(torch.rand(6, 2), torch.rand(6, 1))
    for clone in (pickle.loads(pickle.dumps(gp)), copy.deepcopy(gp)):
        assert torch.equal(clone.train_x, gp.train_x) and torch.equal(clone.train_y, gp.train_y)
        for k, v in gp.state_dict().items():
            assert torch.equal(clone.state_dict()[k], v)
        assert isinstance(clone.kernel, R.SqExp)


def test_gp_symbols_in_the_abi():
    from pytorch_generative_b200 import _build, _lib

    _build.build(verbose=False)
    lib = _lib.load()
    for sym in ("pg_gemm_f64", "pg_gp_potrf", "pg_gp_trsm"):
        assert sym in _lib.EXPORTED_SYMBOLS and hasattr(lib, sym)
    assert _lib.launch_count() >= 0


def _stand_in_reference(tmp_path, with_gp):
    pkg = tmp_path / "pytorch_generative"
    (pkg / "models" / "autoregressive").mkdir(parents=True)
    (pkg / "nn").mkdir()
    (pkg / "__init__.py").write_text("from pytorch_generative import models, nn\n")
    nn_names = ["CausalConv2d", "GatedActivation", "NCHWLayerNorm", "CausalAttention", "LinearCausalAttention"]
    (pkg / "nn" / "__init__.py").write_text("".join(f"class {n}:\n    pass\n" for n in nn_names) +
                                            "def image_positional_encoding(shape):\n    pass\n")
    mods = {"pixel_cnn": "PixelCNN", "gated_pixel_cnn": "GatedPixelCNN", "pixel_snail": "PixelSNAIL",
            "image_gpt": "ImageGPT"}
    for mod, cls in mods.items():
        (pkg / "models" / "autoregressive" / f"{mod}.py").write_text(f"class {cls}:\n    pass\n")
    imports = "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items())
    (pkg / "models" / "autoregressive" / "__init__.py").write_text(imports)
    if with_gp:  # as in the reference: the module exists, models/__init__.py does not export it
        (pkg / "models" / "gaussian_process.py").write_text("class GaussianProcess:\n    pass\n")
    (pkg / "models" / "__init__.py").write_text("from pytorch_generative.models import autoregressive\n" + imports)


@pytest.mark.parametrize("with_gp", [True, False])
def test_overlay_binds_gaussian_process_in_its_module_only(tmp_path, with_gp):
    _stand_in_reference(tmp_path, with_gp)
    sys.path.insert(0, str(tmp_path))
    try:
        import importlib

        import pytorch_generative as ref

        from pytorch_generative_b200 import models, overlay

        mod = importlib.import_module("pytorch_generative.models.gaussian_process") if with_gp else None
        orig = mod.GaussianProcess if with_gp else None
        bound = overlay.install()
        try:
            assert len(bound) == 14 + with_gp
            assert ("pytorch_generative.models.gaussian_process.GaussianProcess" in bound) == with_gp
            assert not hasattr(ref.models, "GaussianProcess")
            if with_gp:
                assert mod.GaussianProcess is models.GaussianProcess
        finally:
            overlay.uninstall()
        if with_gp:
            assert mod.GaussianProcess is orig
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
