"""CPU checks of VeryDeepVAE: the float restatement against the reference fixture (and in float64), the module tree,
state-dict keys, shapes, parameter order and init bits (the reference's decoder kernel size and weight scaling
included), the refusals before any launch, the recipe's signature, the overlay binding and pickle / deepcopy."""

import copy
import inspect
import os
import pickle
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _vd_vae_reference as R  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vd_vae.pt")


@pytest.fixture(scope="module")
def fixture():
    return R.load_fixture(GOLD)


def _model(case):
    from pytorch_generative_b200.models import vd_vae

    kwargs = dict(case["kwargs"])
    if case["stacks"] is not None:
        kwargs["stack_configs"] = [vd_vae.StackConfig(e, d) for e, d in case["stacks"]]
    torch.manual_seed(case["seed"])
    return vd_vae.VeryDeepVAE(**kwargs)


def _cfg(case):
    from pytorch_generative_b200.models import vd_vae

    stacks = case["stacks"] or [(c.n_encoder_blocks, c.n_decoder_blocks) for c in vd_vae.DEFAULT_MODEL]
    return case["kwargs"].get("input_resolution", 32), stacks, case["kwargs"].get("latent_channels", 4)


@pytest.mark.parametrize("name", ["default_32", "rgb_16"])
def test_restatement_matches_the_reference(fixture, name):
    case = fixture[name]
    cfg = _cfg(case)
    logits, kl = R.forward(case["state"], case["x"], cfg, case["eps"])
    torch.testing.assert_close(logits, case["logits"], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(kl, case["kl"], rtol=1e-5, atol=1e-4)
    g, _, _, loss = R.grads(case["state"], case["x"], cfg, case["eps"], torch.float32)
    torch.testing.assert_close(loss.float(), case["losses"]["loss"], rtol=1e-5, atol=1e-4)
    for k, ref in case["grads"].items():
        torch.testing.assert_close(g[k], ref, rtol=1e-4, atol=1e-4 * max(1.0, ref.abs().max().item()), msg=k)
    s = R.sample(case["state"], cfg, case["x"].shape[0], case["sample_eps"])
    torch.testing.assert_close(s, case["sample_logits"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", ["default_32", "rgb_16"])
def test_restatement_in_float64(fixture, name):
    case = fixture[name]
    g64, logits64, kl64, _ = R.grads(case["state"], case["x"], _cfg(case), case["eps"])
    torch.testing.assert_close(logits64.float(), case["logits"], rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(kl64.float(), case["kl"], rtol=1e-3, atol=1e-2)
    for k, ref in case["grads"].items():
        scale = max(1e-6, ref.abs().max().item())
        assert (g64[k].float() - ref).abs().max().item() <= 1e-3 * scale, k


@pytest.mark.parametrize("name", ["default_32", "rgb_16"])
def test_keys_shapes_order_and_init_bits(fixture, name):
    case = fixture[name]
    model = _model(case)
    state = model.state_dict()
    ref = case["state_init"]
    assert list(state) == list(ref)
    for k, v in ref.items():
        assert state[k].shape == v.shape, k
        assert torch.equal(state[k], v), f"init bits of {k}"
    assert [n for n, _ in model.named_parameters()] == list(ref)  # no buffers before the first forward


def test_decoder_kernel_size_follows_the_encoder_loop():
    from pytorch_generative_b200.models import VeryDeepVAE
    from pytorch_generative_b200.models.vd_vae import StackConfig

    model = VeryDeepVAE()  # six stacks down to 1x1: the encoder loop ends with kernel size 1
    for stack in model._decoder:
        for block in stack._topdowns:
            assert block._out._net[3].kernel_size == (1, 1) and block._out._net[3].padding == (0, 0)
            assert block._prior._net[3].kernel_size == (3, 3) and block._posterior._net[3].padding == (1, 1)
    model = VeryDeepVAE(1, 1, 16, [StackConfig(1, 1), StackConfig(1, 1)])  # ends at 8x8: 3x3 everywhere
    assert all(b._out._net[3].kernel_size == (3, 3) for s in model._decoder for b in s._topdowns)


def test_recipe_widths_and_parameter_count():
    from pytorch_generative_b200 import recipes
    from pytorch_generative_b200.models import VeryDeepVAE
    from pytorch_generative_b200.models.vd_vae import StackConfig

    model = VeryDeepVAE(1, 1, 32, [StackConfig(3, 5), StackConfig(3, 5), StackConfig(2, 4), StackConfig(2, 3),
                                   StackConfig(2, 2), StackConfig(1, 1)], latent_channels=16, hidden_channels=64,
                        bottleneck_channels=32)
    assert sum(p.numel() for p in model.parameters()) == 1364705
    convs = [m for m in model.modules() if isinstance(m, torch.nn.Conv2d)]
    assert len(convs) == 314 and sum(c.kernel_size == (3, 3) for c in convs) == 101  # 100 bottleneck 3x3 + _input
    sig = inspect.signature(recipes.reproduce_vd_vae)
    assert list(sig.parameters) == ["n_epochs", "batch_size", "log_dir", "n_gpus", "device_id", "debug_loader"]
    assert sig.parameters["n_epochs"].default == 500 and sig.parameters["batch_size"].default == 128


def test_refusals_before_any_launch():
    from pytorch_generative_b200.models import VeryDeepVAE
    from pytorch_generative_b200.models.vd_vae import BottleneckBlock, StackConfig, TopDownBlock

    with pytest.raises(RuntimeError, match="CUDA"):
        VeryDeepVAE()(torch.zeros(1, 1, 32, 32))
    with pytest.raises(NotImplementedError):
        BottleneckBlock(4, 4, 2)(torch.zeros(1, 4, 2, 2))
    with pytest.raises(NotImplementedError):
        TopDownBlock(4, 1, 2, 3)(torch.zeros(1, 4, 2, 2))
    odd = VeryDeepVAE(1, 1, 6, [StackConfig(1, 1)] * 3)  # 6 -> 3 -> 1: unpooling 1 gives 2, not 3
    with pytest.raises(ValueError, match="even"):
        odd._check_resolutions()
    VeryDeepVAE(1, 1, 16, [StackConfig(1, 1)] * 5)._check_resolutions()


def test_overlay_binds_vd_vae_only_where_the_reference_has_it(tmp_path):
    from pytorch_generative_b200 import overlay

    assert overlay._OPTIONAL_MODEL_NAMES["VeryDeepVAE"] == "vae.vd_vae"
    for with_module in (True, False):
        root = tmp_path / ("with" if with_module else "without")
        pkg = root / "pytorch_generative"
        (pkg / "models" / "vae").mkdir(parents=True)
        (pkg / "models" / "autoregressive").mkdir()
        (pkg / "nn").mkdir()
        (pkg / "__init__.py").write_text("from pytorch_generative import models, nn\n")
        (pkg / "nn" / "__init__.py").write_text("".join(f"{n} = None\n" for n in overlay._NN_NAMES))
        names = list(overlay._MODEL_NAMES) + (["VeryDeepVAE"] if with_module else [])
        (pkg / "models" / "__init__.py").write_text("".join(f"{n} = None\n" for n in names))
        for cls, mod in overlay._MODEL_NAMES.items():
            (pkg / "models" / "autoregressive" / f"{mod}.py").write_text(f"{cls} = None\n")
        if with_module:
            (pkg / "models" / "vae" / "vd_vae.py").write_text("VeryDeepVAE = None\n")
        sys.path.insert(0, str(root))
        try:
            for m in [m for m in sys.modules if m.startswith("pytorch_generative") and not m.startswith(
                    "pytorch_generative_b200")]:
                del sys.modules[m]
            from pytorch_generative_b200.models import VeryDeepVAE

            bound = overlay.install()
            import pytorch_generative as ref

            try:
                has = "pytorch_generative.models.VeryDeepVAE" in bound
                assert has == with_module
                if with_module:
                    import pytorch_generative.models.vae.vd_vae as ref_mod

                    assert ref.models.VeryDeepVAE is VeryDeepVAE and ref_mod.VeryDeepVAE is VeryDeepVAE
            finally:
                overlay.uninstall()
        finally:
            sys.path.remove(str(root))
            for m in [m for m in sys.modules if m.startswith("pytorch_generative") and not m.startswith(
                    "pytorch_generative_b200")]:
                del sys.modules[m]


def test_pickle_and_deepcopy():
    from pytorch_generative_b200.models import VeryDeepVAE

    torch.manual_seed(0)
    model = VeryDeepVAE()
    for clone in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
        a, b = model.state_dict(), clone.state_dict()
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
