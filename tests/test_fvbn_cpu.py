"""FVBN without a GPU: the restatement (tests/_fvbn_reference.py) against the reference's own outputs
(tests/golden/fvbn.pt), the model's constructor, state-dict keys, shapes, parameter order and initial bits, the packed
gradient layout, the refusal to run on CPU tensors, the recipe's signature and the overlay binding of
FullyVisibleBeliefNetwork."""

import inspect
import os
import pickle
import sys

import pytest
import torch

import _fvbn_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "fvbn.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _close(a, b, tol=1e-5):
    return (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())


def test_reference_restatement_matches_the_reference(fixture):
    for name, fx in fixture.items():
        for kind in ("binary", "negative"):
            f = fx[kind]
            logits, loss, grads, x_grad = R.loss_and_grads(fx["state"], f["x"])
            assert _close(logits, f["logits"]), (name, kind)
            assert _close(loss, f["loss"]), (name, kind)
            if f["x_grad"] is None:  # n_dims 1: the input feeds no row
                assert fx["kwargs"]["n_dims"] == 1
            else:
                assert _close(x_grad, f["x_grad"]), (name, kind)
            assert list(grads) == list(f["grads"]), name
            for k, g in f["grads"].items():
                assert _close(grads[k], g), (name, kind, k)
        for kind in ("unconditional", "conditional"):
            s = fx[kind]
            start = s["conditioned_on"] if s["conditioned_on"] is not None else -torch.ones_like(s["sample"])
            got = R.sample(fx["state"], start, R.uniform_sample_fn(s["uniforms"]))
            assert torch.equal(got, s["sample"]), (name, kind)


def test_constructor_keys_shapes_order_and_init_bits_match_the_reference(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture.items():
        D = fx["kwargs"]["n_dims"]
        torch.manual_seed(10 * list(fixture).index(name))
        m = models.FullyVisibleBeliefNetwork(**fx["kwargs"])
        assert m.n_dims == D and len(m._net) == D
        assert [k for k, _ in m.named_parameters()] == R.names(D)
        sd = m.state_dict()
        assert list(sd) == list(fx["state_init"]), name
        for k, v in fx["state_init"].items():
            assert sd[k].dtype == v.dtype and sd[k].shape == v.shape and torch.equal(sd[k], v), (name, k)
        for i in range(D):
            assert sd[f"_net.{i}.weight"].shape == (1, max(1, i)) and sd[f"_net.{i}.bias"].shape == (1,)
        m.load_state_dict(fx["state_after"])  # including the _c/_h/_w buffers of an image forward
        assert int(m._c) * int(m._h) * int(m._w) == D
    sig = inspect.signature(models.FullyVisibleBeliefNetwork.__init__)
    assert [(k, v.default) for k, v in sig.parameters.items()][1:] == [
        ("n_dims", inspect.Parameter.empty), ("sample_fn", None)]
    fn = lambda logits: logits
    assert models.FullyVisibleBeliefNetwork(4, sample_fn=fn)._sample_fn is fn


@pytest.mark.parametrize("D", [1, 2, 3, 37, 784])
def test_packed_offsets(D):
    from pytorch_generative_b200.models import fvbn

    offsets, lengths, total = fvbn.packed_offsets(D)
    assert (offsets, total) == R.offsets(D)
    assert lengths == [max(1, i) for i in range(D)]
    assert offsets[0] == 0 and total == offsets[-1] + lengths[-1]
    assert all(offsets[i + 1] == offsets[i] + lengths[i] for i in range(D - 1))
    # the gradient views of one [T + D] buffer: a [1, len] view per weight, a [1] view per bias, parameters() order
    layout = fvbn.ParamTable(D)
    buf = torch.arange(total + D, dtype=torch.float32)
    grads = layout.grads(buf)
    assert len(grads) == 2 * D
    for i in range(D):
        w, b = grads[2 * i], grads[2 * i + 1]
        assert w.shape == (1, lengths[i]) and w.is_contiguous() and b.shape == (1,)
        assert w.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr()
        assert torch.equal(w[0], buf[offsets[i]: offsets[i] + lengths[i]]) and b.item() == total + i


def test_forward_and_sample_refuse_cpu_tensors():
    from pytorch_generative_b200 import models

    m = models.FullyVisibleBeliefNetwork(16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 16))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.sample(conditioned_on=-torch.ones(2, 1, 4, 4))


def test_the_table_refuses_parameters_the_kernels_cannot_read():
    """The table is built only from CUDA fp32 contiguous rows of max(1, i) (weights) and 1 (biases) elements."""
    from pytorch_generative_b200 import models
    from pytorch_generative_b200.models import fvbn

    m = models.FullyVisibleBeliefNetwork(4)
    layout = fvbn.ParamTable(4)
    params = m._params()
    with pytest.raises(RuntimeError, match="contiguous fp32 tensors on one CUDA device"):
        layout.table(params[0::2], params[1::2])  # CPU parameters
    assert not layout._tables


def test_runtime_caches_stay_out_of_pickles():
    from pytorch_generative_b200 import models

    m = models.FullyVisibleBeliefNetwork(8)
    m.__dict__["_fvbn_table"] = object()  # not picklable
    m.__dict__["_fvbn_sampler"] = {"graph": object()}
    clone = pickle.loads(pickle.dumps(m))
    assert "_fvbn_table" not in clone.__dict__ and "_fvbn_sampler" not in clone.__dict__
    for k, v in m.state_dict().items():
        assert torch.equal(clone.state_dict()[k], v)


def test_reproduce_fvbn_signature():
    from pytorch_generative_b200 import recipes
    from pytorch_generative_b200.models import fvbn

    sig = inspect.signature(recipes.reproduce_fvbn)
    assert {k: v.default for k, v in sig.parameters.items()} == dict(
        n_epochs=50, batch_size=512, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None)
    assert fvbn.reproduce.__doc__ and "reproduce_fvbn" in inspect.getsource(fvbn.reproduce)
    with pytest.raises(RuntimeError, match="CUDA"):
        recipes.reproduce_fvbn(n_gpus=0, debug_loader=[])


def _stand_in_reference(tmp_path, with_fvbn):
    """A stand-in reference package under tmp_path: the four hot-path models, and fvbn.py when asked for."""
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
    if with_fvbn:
        mods["fvbn"] = "FullyVisibleBeliefNetwork"
        (pkg / "models" / "autoregressive" / "fvbn.py").write_text(
            "class FullyVisibleBeliefNetwork:\n    pass\n\ndef reproduce():\n    from pytorch_generative import models\n"
            "    return models.FullyVisibleBeliefNetwork(n_dims=784)\n")
    (pkg / "models" / "autoregressive" / "__init__.py").write_text(
        "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items()))
    (pkg / "models" / "__init__.py").write_text(
        "from pytorch_generative.models import autoregressive\n" +
        "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items()))


@pytest.mark.parametrize("with_fvbn", [True, False])
def test_overlay_binds_fvbn_only_where_the_reference_has_it(tmp_path, with_fvbn):
    """install() binds FullyVisibleBeliefNetwork in both namespaces where the stand-in has fvbn.py, so the reference's
    `reproduce` builds this package's class; without fvbn.py the name is not bound.  uninstall() restores the names."""
    _stand_in_reference(tmp_path, with_fvbn)
    sys.path.insert(0, str(tmp_path))
    try:
        import pytorch_generative as ref

        from pytorch_generative_b200 import models, overlay

        orig = getattr(ref.models, "FullyVisibleBeliefNetwork", None)
        bound = overlay.install()
        try:
            assert ("pytorch_generative.models.FullyVisibleBeliefNetwork" in bound) == with_fvbn
            assert ("pytorch_generative.models.autoregressive.fvbn.FullyVisibleBeliefNetwork" in bound) == with_fvbn
            if with_fvbn:
                from pytorch_generative.models.autoregressive import fvbn as ref_fvbn

                assert ref.models.FullyVisibleBeliefNetwork is models.FullyVisibleBeliefNetwork
                assert ref_fvbn.FullyVisibleBeliefNetwork is models.FullyVisibleBeliefNetwork
                assert isinstance(ref_fvbn.reproduce(), models.FullyVisibleBeliefNetwork)
            else:
                assert not hasattr(ref.models, "FullyVisibleBeliefNetwork")
        finally:
            overlay.uninstall()
        assert getattr(ref.models, "FullyVisibleBeliefNetwork", None) is orig
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
