"""NADE without a GPU: the restatement (tests/_nade_reference.py) against the reference's own outputs
(tests/golden/nade.pt), the model's constructor, parameters and initial bits, the refusal to run on CPU tensors, the
recipe's signature, the checkpoint interval shared by the header and the binding, and the overlay binding of NADE."""

import inspect
import os
import re
import sys

import pytest
import torch

import _nade_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "nade.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _close(a, b, tol=1e-5):
    return (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())


def test_reference_restatement_matches_the_reference(fixture):
    for name, fx in fixture.items():
        for kind in ("binary", "negative"):
            f = fx[kind]
            p, xt, loss, grads, x_grad = R.loss_and_grads(fx["state"], f["x"], f["uniforms"])
            assert _close(p, f["p"]), (name, kind)
            assert torch.equal(xt, f["xt"]), (name, kind)
            assert _close(loss, f["loss"]), (name, kind)
            assert _close(x_grad, f["x_grad"]), (name, kind)
            for k, g in f["grads"].items():
                assert _close(grads[k], g), (name, kind, k)
        assert bool((fx["negative"]["x_grad"][fx["negative"]["x"] < 0] == 0).all()), name
        for kind in ("unconditional", "conditional"):
            s = fx[kind]
            start = s["conditioned_on"] if s["conditioned_on"] is not None else -torch.ones_like(s["sample"])
            assert torch.equal(R.sample(fx["state"], start, s["uniforms"]), s["sample"]), (name, kind)


def test_hidden_preactivations_follow_the_reference_arithmetic(fixture):
    """The a_d that the loop of `forward` consumes are the ones `hidden_preactivations` restates (bit for bit)."""
    fx = fixture["image_64_32"]
    f = fx["negative"]
    p = {k: fx["state"][k] for k in R.PARAMS}
    a = R.hidden_preactivations(p, f["xt"])
    n = f["x"].shape[0]
    z = (torch.relu(a) * p["_h_W"].unsqueeze(0)).sum(-1) + p["_h_b"]
    assert a.shape == (n, 64, 32)
    assert torch.equal(a[:, 0], p["_in_b"].expand(n, -1))
    assert _close(torch.sigmoid(z), f["p"].view(n, -1))


def test_constructor_parameters_and_init_bits_match_the_reference(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture.items():
        torch.manual_seed(10 * list(fixture).index(name))
        m = models.NADE(**fx["kwargs"])
        assert [k for k, _ in m.named_parameters()] == list(R.PARAMS)
        sd = m.state_dict()
        assert list(sd) == list(fx["state_init"]), name
        for k, v in fx["state_init"].items():
            assert sd[k].dtype == v.dtype and torch.equal(sd[k], v), (name, k)
        m.load_state_dict(fx["state_after"])  # including the _c/_h/_w buffers of an image forward
        if "_c" in fx["state_after"]:
            assert int(m._c) * int(m._h) * int(m._w) == fx["kwargs"]["input_dim"]
    sig = inspect.signature(models.NADE.__init__)
    assert [(k, v.default) for k, v in sig.parameters.items()][1:] == [
        ("input_dim", inspect.Parameter.empty), ("hidden_dim", inspect.Parameter.empty), ("sample_fn", None)]
    fn = lambda logits: logits
    assert models.NADE(4, 2, sample_fn=fn)._sample_fn is fn  # stored (and, as in the reference, never called)


def test_forward_and_sample_refuse_cpu_tensors():
    from pytorch_generative_b200 import models

    m = models.NADE(16, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 16))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.sample(conditioned_on=-torch.ones(2, 16))


def test_reproduce_nade_signature():
    from pytorch_generative_b200 import recipes
    from pytorch_generative_b200.models import nade

    sig = inspect.signature(recipes.reproduce_nade)
    assert {k: v.default for k, v in sig.parameters.items()} == dict(
        n_epochs=50, batch_size=512, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None)
    assert nade.reproduce.__doc__ and "reproduce_nade" in inspect.getsource(nade.reproduce)
    with pytest.raises(RuntimeError, match="CUDA"):
        recipes.reproduce_nade(n_gpus=0, debug_loader=[])


def test_checkpoint_interval_matches_the_header():
    from pytorch_generative_b200 import _lib

    text = open(os.path.join(ROOT, "include", "pg_b200.h")).read()
    assert int(re.search(r"#define PG_NADE_CHUNK (\d+)", text).group(1)) == _lib.NADE_CHUNK


def test_overlay_binds_nade_where_the_reference_has_it(tmp_path):
    """A stand-in reference with models/autoregressive/nade.py: install() binds NADE in both namespaces, so the
    reference's `reproduce` (which builds `models.NADE(...)`) gets this package's class; uninstall() restores it."""
    pkg = tmp_path / "pytorch_generative"
    (pkg / "models" / "autoregressive").mkdir(parents=True)
    (pkg / "nn").mkdir()
    (pkg / "__init__.py").write_text("from pytorch_generative import models, nn\n")
    nn_names = ["CausalConv2d", "GatedActivation", "NCHWLayerNorm", "CausalAttention", "LinearCausalAttention"]
    (pkg / "nn" / "__init__.py").write_text("".join(f"class {n}:\n    pass\n" for n in nn_names) +
                                            "def image_positional_encoding(shape):\n    pass\n")
    mods = {"pixel_cnn": "PixelCNN", "gated_pixel_cnn": "GatedPixelCNN", "pixel_snail": "PixelSNAIL",
            "image_gpt": "ImageGPT", "nade": "NADE"}
    for mod, cls in mods.items():
        (pkg / "models" / "autoregressive" / f"{mod}.py").write_text(f"class {cls}:\n    pass\n")
    (pkg / "models" / "autoregressive" / "nade.py").write_text(
        "class NADE:\n    pass\n\ndef reproduce():\n    from pytorch_generative import models\n"
        "    return models.NADE(input_dim=784, hidden_dim=500)\n")
    (pkg / "models" / "autoregressive" / "__init__.py").write_text(
        "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items()))
    (pkg / "models" / "__init__.py").write_text(
        "from pytorch_generative.models import autoregressive\n" +
        "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items()))
    sys.path.insert(0, str(tmp_path))
    try:
        import pytorch_generative as ref
        from pytorch_generative.models.autoregressive import nade as ref_nade

        from pytorch_generative_b200 import models, overlay

        orig = ref.models.NADE
        bound = overlay.install()
        try:
            assert ref.models.NADE is models.NADE and ref_nade.NADE is models.NADE
            assert "pytorch_generative.models.NADE" in bound
            assert "pytorch_generative.models.autoregressive.nade.NADE" in bound
            assert "pytorch_generative.models.MADE" not in bound  # the stand-in has no made.py
            assert isinstance(ref_nade.reproduce(), models.NADE)
        finally:
            overlay.uninstall()
        assert ref.models.NADE is orig and ref_nade.NADE is orig
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
