"""VQ-VAE, VQ-VAE-2 and VectorQuantizer without a GPU: the restatement (tests/_vq_vae_reference.py) against the
reference's own outputs, gradients and buffers (tests/golden/vq_vae.pt), a float64 restatement, the constructors' keys,
shapes, order and init bits of parameters and buffers, the refusals, the recipes' signatures, the overlay, pickling and
deepcopy, sampling's refusal and CIFAR-10's normalisation."""

import copy
import inspect
import os
import pickle
import sys

import pytest
import torch

import _vq_vae_reference as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vq_vae.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _build(fx):
    from pytorch_generative_b200 import models, nn

    if fx["cls"] == "VectorQuantizer":
        return nn.VectorQuantizer(**fx["kwargs"])
    return getattr(models, fx["cls"])(**fx["kwargs"])


def test_reference_restatement_matches_the_reference(fixture):
    """In fp32 the restatement performs the reference's operations in the reference's order: equal bit for bit, the
    quantizers' inputs, indices and updated buffers included."""
    for name, fx in fixture.items():
        out, losses, grads, found = R.run(fx)
        assert torch.equal(out, fx["outputs"]), name
        if fx["cls"] == "VectorQuantizer":
            assert torch.equal(losses, fx["vq_loss"]) and torch.equal(grads.pop("x"), fx["x_grad"])
        else:
            for k, v in fx["losses"].items():
                assert torch.equal(losses[k], v), (name, k)
        assert list(grads) == list(fx["grads"]), name
        for k, g in fx["grads"].items():
            assert torch.equal(grads[k], g), (name, k)
        for k, s in fx["vq_inputs"].items():
            assert torch.equal(found[k]["input"], s["input"]) and torch.equal(found[k]["idx"], s["idx"]), (name, k)
            if found[k]["buffers"] is not None:
                for b, n in zip(found[k]["buffers"], ("_cluster_size", "_embedding_avg", "_embedding")):
                    assert torch.equal(b, fx["buffers"][f"{k}.{n}"]), (name, k, n)
            else:  # eval() or no EMA: the buffers are the ones loaded
                for n in ("_cluster_size", "_embedding_avg", "_embedding"):
                    if f"{k}.{n}" in fx["buffers"]:
                        assert torch.equal(fx["buffers"][f"{k}.{n}"], fx["state"][f"{k}.{n}"]), (name, k, n)
            assert s["margin"].min() >= 0.05, (name, k)


def test_float64_restatement_agrees_with_the_reference(fixture):
    for name, fx in fixture.items():
        out, losses, grads, found = R.run(fx, torch.float64)
        for k, s in fx["vq_inputs"].items():
            assert torch.equal(found[k]["idx"], s["idx"]), (name, k)
        assert torch.allclose(out.float(), fx["outputs"], rtol=1e-4, atol=1e-4), name
        for k, g in fx["grads"].items():
            assert torch.allclose(grads[k].float(), g, rtol=1e-3, atol=1e-4), (name, k)


def test_constructor_keys_shapes_order_and_init_bits_match_the_reference(fixture):
    from pytorch_generative_b200 import models
    from pytorch_generative_b200.models import vae

    for name, fx in fixture.items():
        torch.manual_seed(fx["seed"])
        m = _build(fx)
        assert [k for k, _ in m.named_parameters()] == list(fx["grads"]), name
        assert [k for k, _ in m.named_buffers()] == [k for k in fx["state_init"] if k in fx["buffers"]], name
        sd = m.state_dict()
        assert list(sd) == list(fx["state_init"]), name
        for k, v in fx["state_init"].items():
            assert sd[k].dtype == v.dtype and sd[k].shape == v.shape and torch.equal(sd[k], v), (name, k)
        if fx["cls"] != "VectorQuantizer":
            assert all(isinstance(q, vae.Quantizer) for n, q in m.named_children() if n.startswith("_quantizer"))
    # the recipe sizes
    assert [(k, v.default) for k, v in inspect.signature(models.VectorQuantizedVAE.__init__).parameters.items()][1:] == [
        ("in_channels", 1), ("out_channels", 1), ("hidden_channels", 128), ("n_residual_blocks", 2),
        ("residual_channels", 32), ("n_embeddings", 128), ("embedding_dim", 16), ("sample_fn", None)]
    assert (list(inspect.signature(models.VectorQuantizedVAE2.__init__).parameters)
            == list(inspect.signature(models.VectorQuantizedVAE.__init__).parameters))
    assert issubclass(models.VectorQuantizedVAE, models.VariationalAutoEncoder)
    assert issubclass(models.VectorQuantizedVAE2, models.VariationalAutoEncoder)


def test_refusals():
    """CPU tensors, non-fp32 inputs, odd strides and the reference's channel assertion raise before any launch."""
    from pytorch_generative_b200 import losses, models, nn

    m = models.VectorQuantizedVAE(3, 3, 8, 1, 8, 4, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 3, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        models.VectorQuantizedVAE2(3, 3, 8, 1, 8, 4, 4)(torch.zeros(2, 3, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        nn.VectorQuantizer(4, 4)(torch.zeros(2, 4, 3, 3))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m._quantizer(torch.zeros(2, 8, 2, 2))
    with pytest.raises(AssertionError, match="embedding_dim"):
        nn.VectorQuantizer(4, 4)(torch.zeros(2, 3, 3, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        losses.mse_loss(torch.zeros(2, 3), torch.zeros(2, 3))
    with pytest.raises(ValueError, match="differ"):
        losses.mse_loss(torch.zeros(2, 3), torch.zeros(3, 2))


@pytest.mark.parametrize("cls", ["VectorQuantizedVAE", "VectorQuantizedVAE2"])
def test_sample_raises_as_the_reference(cls):
    from pytorch_generative_b200 import models

    m = getattr(models, cls)(3, 3, 8, 1, 8, 4, 4)
    m._register_shape(3, 8, 8)
    with pytest.raises(NotImplementedError, match="does not support sampling"):
        m.sample(2)


@pytest.mark.parametrize("use_ema", [True, False])
def test_pickle_and_deepcopy_keep_the_buffers(use_ema):
    from pytorch_generative_b200 import models

    torch.manual_seed(3)
    m = models.VectorQuantizedVAE(3, 3, 8, 1, 8, 4, 4)
    m._quantizer._net[1]._use_ema = use_ema
    with torch.no_grad():
        m._quantizer._net[1]._cluster_size.uniform_()
    for clone in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert list(clone.state_dict()) == list(m.state_dict())
        for k, v in m.state_dict().items():
            assert torch.equal(clone.state_dict()[k], v), k
        assert clone._quantizer._net[1]._use_ema == use_ema


@pytest.mark.parametrize("name, weight", [("vq_vae", "vq_vae_loss"), ("vq_vae_2", "vq_vae_2_loss")])
def test_recipe_signatures(name, weight):
    from pytorch_generative_b200 import losses, models, recipes

    fn = getattr(recipes, f"reproduce_{name}")
    sig = inspect.signature(fn)
    assert {k: v.default for k, v in sig.parameters.items()} == dict(
        n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None)
    src = inspect.getsource(fn)
    assert "n_embeddings=512, embedding_dim=64" in src and "2e-4, 0.999977" in src and '"normalize": True' in src
    assert f"losses.{weight}" in src and 'dataset="cifar10"' in src
    assert ("residual_channels=32" if name == "vq_vae" else "residual_channels=64") in src
    mod = getattr(models, name)
    assert mod.reproduce.__doc__ and f"reproduce_{name}" in inspect.getsource(mod.reproduce)
    assert list(inspect.signature(getattr(losses, weight)).parameters) == ["x", "_", "preds"]
    assert "0.25 * vq_loss" in inspect.getsource(losses.vq_vae_2_loss)
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(n_gpus=0, debug_loader=[])
    from pytorch_generative_b200 import datasets

    params = list(inspect.signature(datasets.get_cifar10_loaders).parameters)
    assert params == ["batch_size", "device", "download", "normalize"]
    assert inspect.signature(datasets.get_cifar10_loaders).parameters["normalize"].default is False


def test_normalize_agrees_with_the_reference_formula():
    """DeviceTransform's normalisation of a uint8 batch equals ToTensor then Normalize((0.4914, 0.4822, 0.4465),
    (0.2023, 0.1994, 0.2010)), written out as torchvision computes it: (x / 255 - mean) / std per channel."""
    from pytorch_generative_b200 import datasets

    images = torch.randint(0, 256, (5, 3, 4, 6), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    got = next(iter(datasets.DeviceTransform([(images, torch.zeros(5))], "cpu", normalize=True)))[0]
    x = images.float() / 255
    mean = torch.tensor([0.4914, 0.4822, 0.4465]).view(-1, 1, 1)
    std = torch.tensor([0.2023, 0.1994, 0.2010]).view(-1, 1, 1)
    want = torch.stack([x[i].sub(mean).div(std) for i in range(5)])
    assert torch.equal(got, want)
    plain = next(iter(datasets.DeviceTransform([(images, torch.zeros(5))], "cpu")))[0]
    assert torch.equal(plain, x)


def _stand_in_reference(tmp_path, with_vq):
    """A stand-in reference package: the four hot-path models and, when asked for, vae/vq_vae.py, vae/vq_vae_2.py and
    VectorQuantizer in nn/utils.py and nn/__init__.py."""
    pkg = tmp_path / "pytorch_generative"
    (pkg / "models" / "autoregressive").mkdir(parents=True)
    (pkg / "nn").mkdir()
    (pkg / "__init__.py").write_text("from pytorch_generative import models, nn\n")
    nn_names = ["CausalConv2d", "GatedActivation", "NCHWLayerNorm", "CausalAttention", "LinearCausalAttention"]
    nn_init = "".join(f"class {n}:\n    pass\n" for n in nn_names) + "def image_positional_encoding(shape):\n    pass\n"
    if with_vq:
        (pkg / "nn" / "utils.py").write_text("class VectorQuantizer:\n    pass\n")
        nn_init += "from pytorch_generative.nn.utils import VectorQuantizer\n"
    (pkg / "nn" / "__init__.py").write_text(nn_init)
    mods = {"pixel_cnn": "PixelCNN", "gated_pixel_cnn": "GatedPixelCNN", "pixel_snail": "PixelSNAIL",
            "image_gpt": "ImageGPT"}
    for mod, cls in mods.items():
        (pkg / "models" / "autoregressive" / f"{mod}.py").write_text(f"class {cls}:\n    pass\n")
    imports = "".join(f"from pytorch_generative.models.autoregressive.{m} import {c}\n" for m, c in mods.items())
    (pkg / "models" / "autoregressive" / "__init__.py").write_text(imports)
    if with_vq:
        (pkg / "models" / "vae").mkdir()
        for mod, cls in (("vq_vae", "VectorQuantizedVAE"), ("vq_vae_2", "VectorQuantizedVAE2")):
            (pkg / "models" / "vae" / f"{mod}.py").write_text(
                f"class {cls}:\n    pass\n\ndef reproduce():\n    from pytorch_generative import models\n"
                f"    return models.{cls}(3, 3, 8, 1, 8, 4, 4)\n")
            imports += f"from pytorch_generative.models.vae.{mod} import {cls}\n"
    (pkg / "models" / "__init__.py").write_text("from pytorch_generative.models import autoregressive\n" + imports)


@pytest.mark.parametrize("with_vq", [True, False])
def test_overlay_binds_the_vq_names_only_where_the_reference_has_them(tmp_path, with_vq):
    _stand_in_reference(tmp_path, with_vq)
    sys.path.insert(0, str(tmp_path))
    try:
        import pytorch_generative as ref

        from pytorch_generative_b200 import models, nn, overlay

        bound = overlay.install()
        try:
            for cls, mod in (("VectorQuantizedVAE", "vq_vae"), ("VectorQuantizedVAE2", "vq_vae_2")):
                assert (f"pytorch_generative.models.{cls}" in bound) == with_vq
                assert (f"pytorch_generative.models.vae.{mod}.{cls}" in bound) == with_vq
            assert ("pytorch_generative.nn.VectorQuantizer" in bound) == with_vq
            assert ("pytorch_generative.nn.utils.VectorQuantizer" in bound) == with_vq
            assert len(bound) == 14 + 6 * with_vq
            if with_vq:
                from pytorch_generative.models.vae import vq_vae as ref_vq, vq_vae_2 as ref_vq2
                from pytorch_generative.nn import utils as ref_utils

                assert ref.models.VectorQuantizedVAE is models.VectorQuantizedVAE
                assert ref.nn.VectorQuantizer is nn.VectorQuantizer and ref_utils.VectorQuantizer is nn.VectorQuantizer
                assert isinstance(ref_vq.reproduce(), models.VectorQuantizedVAE)
                assert isinstance(ref_vq2.reproduce(), models.VectorQuantizedVAE2)
            else:
                assert not hasattr(ref.nn, "VectorQuantizer") and not hasattr(ref.models, "VectorQuantizedVAE")
        finally:
            overlay.uninstall()
        if with_vq:
            from pytorch_generative.models.vae import vq_vae as ref_vq
            from pytorch_generative.nn import utils as ref_utils

            assert ref.models.VectorQuantizedVAE is not models.VectorQuantizedVAE
            assert ref_vq.VectorQuantizedVAE is not models.VectorQuantizedVAE
            assert ref.nn.VectorQuantizer is not nn.VectorQuantizer and ref_utils.VectorQuantizer is not nn.VectorQuantizer
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
