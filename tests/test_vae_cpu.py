"""VAE and BetaVAE without a GPU: the restatement (tests/_vae_reference.py) against the reference's own outputs
(tests/golden/vae.pt), the constructors, state-dict keys, shapes, parameter order and initial bits, the refusal to run
on CPU tensors, the odd-stride error, the recipes' signatures and the overlay binding of both models."""

import inspect
import pickle
import os
import sys

import pytest
import torch

import _vae_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "vae.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _build(fx):
    from pytorch_generative_b200 import models

    return getattr(models, fx["cls"])(**fx["kwargs"])


def test_reference_restatement_matches_the_reference(fixture):
    """In fp32 the restatement performs the reference's operations in the reference's order: equal bit for bit."""
    for name, fx in fixture.items():
        kw = fx["kwargs"]
        logits, kl, losses, grads = R.loss_and_grads(fx["state"], fx["x"], fx["eps"], kw["latent_channels"],
                                                     kw.get("beta"))
        assert torch.equal(logits, fx["logits"]) and torch.equal(kl, fx["kl"]), name
        for k, v in fx["losses"].items():
            assert torch.equal(losses[k], v), (name, k)
        assert list(grads) == list(fx["grads"]), name
        for k, g in fx["grads"].items():
            assert torch.equal(grads[k], g), (name, k)
        assert torch.equal(R.decode(fx["state"], fx["sample_latents"]), fx["sample_logits"]), name


def test_float64_restatement_agrees_with_the_reference(fixture):
    for name, fx in fixture.items():
        kw = fx["kwargs"]
        logits, kl, losses, grads = R.loss_and_grads(fx["state"], fx["x"], fx["eps"], kw["latent_channels"],
                                                     kw.get("beta"), torch.float64)
        assert torch.allclose(logits.float(), fx["logits"], rtol=1e-4, atol=1e-4), name
        assert torch.allclose(kl.float(), fx["kl"], rtol=1e-4, atol=1e-4), name
        for k, g in fx["grads"].items():
            assert torch.allclose(grads[k].float(), g, rtol=1e-3, atol=1e-4), (name, k)


def test_constructor_keys_shapes_order_and_init_bits_match_the_reference(fixture):
    from pytorch_generative_b200 import models
    from pytorch_generative_b200.models import vae

    for name, fx in fixture.items():
        torch.manual_seed(fx["seed"])
        m = _build(fx)
        assert [k for k, _ in m.named_parameters()] == list(fx["grads"]), name
        sd = m.state_dict()
        assert list(sd) == list(fx["state_init"]), name
        for k, v in fx["state_init"].items():
            assert sd[k].dtype == v.dtype and sd[k].shape == v.shape and torch.equal(sd[k], v), (name, k)
        assert all(isinstance(e, vae.Encoder) for e in m._encoder) and all(isinstance(d, vae.Decoder) for d in m._decoder)
        m.load_state_dict({**fx["state"], **fx["shape_buffers"]})
        assert (int(m._c), int(m._h), int(m._w)) == tuple(fx["x"].shape[1:]), name
    # the recipe sizes: 974,241 parameters, beta = 4
    m = models.VAE(1, 1, 16, [2, 2, 2, 2], 64, 32)
    assert sum(p.numel() for p in m.parameters()) == 974241
    assert models.BetaVAE(1, 1, 4.0, 16, [2, 2, 2, 2], 64, 32)._beta == 4.0
    assert [(k, v.default) for k, v in inspect.signature(models.VAE.__init__).parameters.items()][1:] == [
        ("in_channels", 1), ("out_channels", 1), ("latent_channels", 16), ("strides", [4]), ("hidden_channels", 64),
        ("residual_channels", 32), ("sample_fn", None)]
    assert [(k, v.default) for k, v in inspect.signature(models.BetaVAE.__init__).parameters.items()][1:] == [
        ("in_channels", 1), ("out_channels", 1), ("beta", 4.0), ("latent_channels", 16), ("strides", [4]),
        ("hidden_channels", 64), ("residual_channels", 32), ("sample_fn", None)]
    assert list(inspect.signature(models.VAE.sample).parameters) == ["self", "n_samples"]
    assert issubclass(models.VAE, models.VariationalAutoEncoder) and issubclass(models.BetaVAE, models.VAE)


def test_odd_strides_raise_like_the_reference():
    from pytorch_generative_b200 import models

    with pytest.raises(AssertionError, match="must be even"):
        models.VAE(strides=[3])
    with pytest.raises(AssertionError, match="must be even"):
        models.BetaVAE(strides=[2, 1])


def test_forward_and_sample_refuse_cpu_tensors():
    from pytorch_generative_b200 import models

    m = models.VAE(1, 1, 4, [2], 8, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 1, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m._encoder[0](torch.zeros(2, 1, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.sample(2)  # the shape buffers exist now: the call above recorded them
    with pytest.raises(AttributeError):
        models.VAE(1, 1, 4, [2], 8, 8).sample(2)  # before any forward, as in the reference


def test_pickles_keep_the_state():
    from pytorch_generative_b200 import models

    m = models.BetaVAE(1, 1, 2.0, 4, [2], 8, 8)
    clone = pickle.loads(pickle.dumps(m))
    assert clone._beta == 2.0
    for k, v in m.state_dict().items():
        assert torch.equal(clone.state_dict()[k], v)


@pytest.mark.parametrize("name, epochs, lr, cls", [("vae", 457, "5e-4", "VAE"), ("beta_vae", 500, "1e-3", "BetaVAE")])
def test_recipe_signatures(name, epochs, lr, cls):
    from pytorch_generative_b200 import losses, recipes
    from pytorch_generative_b200 import models

    fn = getattr(recipes, f"reproduce_{name}")
    sig = inspect.signature(fn)
    assert {k: v.default for k, v in sig.parameters.items()} == dict(
        n_epochs=epochs, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None)
    src = inspect.getsource(fn)
    assert f"models.{cls}(" in src and "strides=[2, 2, 2, 2]" in src and lr in src
    assert '"resize_to_32": True' in src and '"dynamically_binarize": True' in src and "losses.vae_elbo" in src
    mod = getattr(models, name)
    assert mod.reproduce.__doc__ and f"reproduce_{name}" in inspect.getsource(mod.reproduce)
    assert list(inspect.signature(losses.vae_elbo).parameters) == ["x", "_", "preds"]
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(n_gpus=0, debug_loader=[])


def _stand_in_reference(tmp_path, with_vae):
    """A stand-in reference package under tmp_path: the four hot-path models and, when asked for, vae/vae.py and
    vae/beta_vae.py inside a namespace package `vae` (no __init__.py, as in the reference)."""
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
    if with_vae:
        (pkg / "models" / "vae").mkdir()
        (pkg / "models" / "vae" / "vae.py").write_text(
            "class VAE:\n    pass\n\ndef reproduce():\n    from pytorch_generative import models\n"
            "    return models.VAE(1, 1, 16, [2, 2, 2, 2], 64, 32)\n")
        (pkg / "models" / "vae" / "beta_vae.py").write_text(
            "from pytorch_generative.models.vae import vae\n\nclass BetaVAE(vae.VAE):\n    pass\n\n"
            "def reproduce():\n    from pytorch_generative import models\n"
            "    return models.BetaVAE(1, 1, 4.0, 16, [2, 2, 2, 2], 64, 32)\n")
        imports += ("from pytorch_generative.models.vae.vae import VAE\n"
                    "from pytorch_generative.models.vae.beta_vae import BetaVAE\n")
    (pkg / "models" / "__init__.py").write_text("from pytorch_generative.models import autoregressive\n" + imports)


@pytest.mark.parametrize("with_vae", [True, False])
def test_overlay_binds_the_vaes_only_where_the_reference_has_them(tmp_path, with_vae):
    """install() binds VAE and BetaVAE in both namespaces where the stand-in has vae/{vae,beta_vae}.py, so the
    reference's `reproduce` builds this package's classes; without them nothing is bound and nothing raises."""
    _stand_in_reference(tmp_path, with_vae)
    sys.path.insert(0, str(tmp_path))
    try:
        import pytorch_generative as ref

        from pytorch_generative_b200 import models, overlay

        bound = overlay.install()
        try:
            for cls, mod in (("VAE", "vae"), ("BetaVAE", "beta_vae")):
                assert (f"pytorch_generative.models.{cls}" in bound) == with_vae
                assert (f"pytorch_generative.models.vae.{mod}.{cls}" in bound) == with_vae
            assert len(bound) == 14 + 4 * with_vae
            if with_vae:
                from pytorch_generative.models.vae import beta_vae as ref_beta
                from pytorch_generative.models.vae import vae as ref_vae

                assert ref.models.VAE is models.VAE and ref_vae.VAE is models.VAE
                assert ref.models.BetaVAE is models.BetaVAE and ref_beta.BetaVAE is models.BetaVAE
                assert isinstance(ref_vae.reproduce(), models.VAE)
                assert isinstance(ref_beta.reproduce(), models.BetaVAE)
            else:
                assert not hasattr(ref.models, "VAE") and not hasattr(ref.models, "BetaVAE")
        finally:
            overlay.uninstall()
        if with_vae:
            from pytorch_generative.models.vae import vae as ref_vae

            assert ref.models.VAE is not models.VAE and ref_vae.VAE is not models.VAE
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]


def test_strided_ops_refuse_settings_off_the_path():
    """groups, dilation, output_padding, padding modes other than zeros and string padding raise NotImplementedError
    before any launch; so does an input too small for the kernel (a ValueError)."""
    from torch import nn

    from pytorch_generative_b200.nn import pm

    x, geom = torch.zeros(2 * 64, 8), pm.Geom(2, 8, 8)
    for conv in (nn.Conv2d(8, 8, 4, 2, 1, groups=2), nn.Conv2d(8, 8, 4, 2, 1, dilation=2),
                 nn.Conv2d(8, 8, 4, 2, 1, padding_mode="reflect"), nn.Conv2d(8, 8, 3, 1, padding="same"),
                 nn.Conv2d(8, 8, 4, (2, 1), 1)):
        with pytest.raises(NotImplementedError):
            pm.conv_strided(x, conv, geom)
    for conv in (nn.ConvTranspose2d(8, 8, 4, 2, 1, output_padding=1), nn.ConvTranspose2d(8, 8, 4, 2, 1, groups=2),
                 nn.ConvTranspose2d(8, 8, 4, 2, 1, dilation=2)):
        with pytest.raises(NotImplementedError):
            pm.conv_transposed(x, conv, geom)
    with pytest.raises(ValueError, match="too small"):
        pm.conv_strided(torch.zeros(2 * 1, 8), nn.Conv2d(8, 8, 4, 2, 1), pm.Geom(2, 1, 1))
    assert pm.strided_geom(nn.Conv2d(8, 8, 4, 2, 1), pm.Geom(2, 7, 7)) == pm.Geom(2, 3, 3)
    assert pm.strided_geom(nn.ConvTranspose2d(8, 8, 4, 2, 1), pm.Geom(2, 3, 3)) == pm.Geom(2, 6, 6)
