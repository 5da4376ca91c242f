"""NICE without a GPU: the restatement (tests/_nice_reference.py) against the reference's own outputs
(tests/golden/nice.pt), the constructors, state-dict keys, shapes, parameter order and initial bits, the odd-width
error, the refusal to run on CPU tensors, the recipe's signature and the overlay binding of NICE in both namespaces."""

import inspect
import pickle
import os
import sys

import pytest
import torch

import _nice_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "nice.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def test_reference_restatement_matches_the_reference(fixture):
    """In fp32 the restatement performs the reference's operations in the reference's order: equal bit for bit."""
    for name, fx in fixture.items():
        z, log_det, losses, grads, x_grad = R.loss_and_grads(fx["state"], fx["x"])
        assert torch.equal(z, fx["z"]) and torch.equal(log_det, fx["log_det_J"]), name
        for k, v in fx["losses"].items():
            assert torch.equal(losses[k], v), (name, k)
        assert list(grads) == list(fx["grads"]), name
        for k, g in fx["grads"].items():
            assert torch.equal(grads[k], g), (name, k)
        assert torch.equal(x_grad, fx["x_grad"]), name
        params = R.params_of(fx["state"])
        assert torch.equal(R.inverse(params, fx["z"]), fx["inverse"]), name
        torch.manual_seed(fx["sample_seed"])
        latents = torch.randn(fx["x"].shape) * 0.7
        assert torch.equal(R.inverse(params, latents), fx["sample"]), name


def test_float64_restatement_agrees_with_the_reference(fixture):
    for name, fx in fixture.items():
        z, log_det, losses, grads, x_grad = R.loss_and_grads(fx["state"], fx["x"], torch.float64)
        assert torch.allclose(z.float(), fx["z"], rtol=1e-5, atol=1e-5), name
        assert torch.allclose(losses["loss"].float(), fx["losses"]["loss"], rtol=1e-5), name
        for k, g in fx["grads"].items():
            assert torch.allclose(grads[k].float(), g, rtol=1e-4, atol=1e-5), (name, k)


def test_constructor_keys_shapes_order_and_init_bits_match_the_reference(fixture):
    from pytorch_generative_b200 import models
    from pytorch_generative_b200.models import nice

    for name, fx in fixture.items():
        kw = fx["kwargs"]
        torch.manual_seed(fx["seed"])
        m = models.NICE(**kw)
        assert [k for k, _ in m.named_parameters()] == R.names(fx["state"])
        sd = m.state_dict()
        assert list(sd) == list(fx["state_init"]), name
        for k, v in fx["state_init"].items():
            assert sd[k].dtype == v.dtype and sd[k].shape == v.shape and torch.equal(sd[k], v), (name, k)
        assert len(m.net) == kw["n_coupling_blocks"] and m.scaling.log_scale.shape == (1, kw["n_features"])
        assert [b.reverse for b in m.net] == [b % 2 == 1 for b in range(kw["n_coupling_blocks"])]
        for b in m.net:
            assert isinstance(b, nice.AdditiveCouplingBlock)
            kinds = [type(l).__name__ for l in b.net]
            assert kinds == ["Linear", "ReLU"] * kw["n_hidden_layers"] + ["Linear"]
        m.load_state_dict(fx["state_after"])  # including the _c/_h/_w buffers of an image forward
        assert int(m._c) * int(m._h) * int(m._w) == kw["n_features"]
    # the recipe size: 49 keys, 19,158,352 parameters
    m = models.NICE(784)
    assert len(m.state_dict()) == 49 and sum(p.numel() for p in m.parameters()) == 19158352
    sig = inspect.signature(models.NICE.__init__)
    assert [(k, v.default) for k, v in sig.parameters.items()][1:] == [
        ("n_features", inspect.Parameter.empty), ("n_coupling_blocks", 4), ("n_hidden_layers", 5),
        ("n_hidden_features", 1000)]
    assert list(inspect.signature(models.NICE.sample).parameters) == ["self", "n_samples", "temp"]
    assert inspect.signature(models.NICE.sample).parameters["temp"].default == 1.0


def test_odd_feature_counts_raise_a_value_error():
    """The coupling halves are D/2 wide: an odd D is refused at forward with a ValueError (the reference fails there with
    a shape error), before any device is involved."""
    from pytorch_generative_b200 import models

    m = models.NICE(7, n_coupling_blocks=2, n_hidden_layers=1, n_hidden_features=4)
    with pytest.raises(ValueError, match="must be even"):
        m(torch.zeros(2, 7))
    with pytest.raises(ValueError, match="must be even"):
        m.net[0](torch.zeros(2, 7))
    with pytest.raises(ValueError, match="features"):
        models.NICE(8, 2, 1, 4)(torch.zeros(2, 10))


def test_forward_inverse_and_sample_refuse_cpu_tensors():
    from pytorch_generative_b200 import models

    m = models.NICE(8, 2, 1, 4)
    for call in (lambda: m(torch.zeros(2, 8)), lambda: m.net[0](torch.zeros(2, 8)), lambda: m.scaling(torch.zeros(2, 8)),
                 lambda: m.scaling.log_det_J()):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m._inverse(torch.zeros(2, 8))
    m._register_shape(1, 2, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.sample(2)


def test_runtime_caches_stay_out_of_pickles():
    from pytorch_generative_b200 import models

    m = models.NICE(8, 2, 1, 4)
    clone = pickle.loads(pickle.dumps(m))
    for k, v in m.state_dict().items():
        assert torch.equal(clone.state_dict()[k], v)


def test_reproduce_nice_signature():
    from pytorch_generative_b200 import losses, recipes
    from pytorch_generative_b200.models import nice

    sig = inspect.signature(recipes.reproduce_nice)
    assert {k: v.default for k, v in sig.parameters.items()} == dict(
        n_epochs=150, batch_size=1024, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None)
    assert nice.reproduce.__doc__ and "reproduce_nice" in inspect.getsource(nice.reproduce)
    assert "dequantize" in inspect.getsource(recipes.reproduce_nice)
    assert "logistic_prior_nll" in inspect.getsource(recipes.reproduce_nice)
    assert list(inspect.signature(losses.logistic_prior_nll).parameters) == ["x", "_", "preds"]
    with pytest.raises(RuntimeError, match="CUDA"):
        recipes.reproduce_nice(n_gpus=0, debug_loader=[])
    # the other recipes keep the binarised data and the BCE loss
    run = inspect.signature(recipes._run).parameters
    assert run["loss_fn"].default is recipes.recipe_loss and run["transform"].default is None


def _stand_in_reference(tmp_path, with_nice):
    """A stand-in reference package under tmp_path: the four hot-path models and, when asked for, flow/nice.py inside a
    namespace package `flow` (no __init__.py, as in the reference)."""
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
    if with_nice:
        (pkg / "models" / "flow").mkdir()
        (pkg / "models" / "flow" / "nice.py").write_text(
            "class NICE:\n    pass\n\ndef reproduce():\n    from pytorch_generative import models\n"
            "    return models.NICE(n_features=784, n_coupling_blocks=4, n_hidden_layers=5, n_hidden_features=1000)\n")
        imports += "from pytorch_generative.models.flow.nice import NICE\n"
    (pkg / "models" / "__init__.py").write_text("from pytorch_generative.models import autoregressive\n" + imports)


@pytest.mark.parametrize("with_nice", [True, False])
def test_overlay_binds_nice_only_where_the_reference_has_it(tmp_path, with_nice):
    """install() binds NICE in both namespaces where the stand-in has flow/nice.py, so the reference's `reproduce` builds
    this package's class; without a flow package the name is not bound and nothing raises.  uninstall() restores."""
    _stand_in_reference(tmp_path, with_nice)
    sys.path.insert(0, str(tmp_path))
    try:
        import pytorch_generative as ref

        from pytorch_generative_b200 import models, overlay

        orig = getattr(ref.models, "NICE", None)
        bound = overlay.install()
        try:
            assert ("pytorch_generative.models.NICE" in bound) == with_nice
            assert ("pytorch_generative.models.flow.nice.NICE" in bound) == with_nice
            assert len(bound) == 14 + 2 * with_nice
            if with_nice:
                from pytorch_generative.models.flow import nice as ref_nice

                assert ref.models.NICE is models.NICE and ref_nice.NICE is models.NICE
                assert isinstance(ref_nice.reproduce(), models.NICE)
            else:
                assert not hasattr(ref.models, "NICE")
        finally:
            overlay.uninstall()
        assert getattr(ref.models, "NICE", None) is orig
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
