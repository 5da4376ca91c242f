"""Mixture models and KDE without a GPU: the restatement (tests/_density_reference.py) against the reference's own
outputs (tests/golden/density.pt), constructors, state-dict keys, shapes, parameter order and init bits, the refusals
(CPU tensors, other dtypes, training data that requires grad), sample() before any forward, the Parzen boundary with a
`<` bug model, the overlay binding and pickle / deepcopy."""

import copy
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import _density_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "density.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def test_fixture_is_small():
    assert os.path.getsize(GOLD) < 1 << 20


def test_mixture_restatement_matches_the_reference(fixture):
    for name, fx in fixture["mixture"].items():
        out, grads, x_grad = R.mixture_loss_and_grads(fx["cls"], fx["state"], fx["x"], fx["cot"])
        assert torch.equal(out, fx["out"]), name
        assert list(grads) == list(fx["grads"]) == R.mixture_names(fx["cls"]), name
        for k, g in fx["grads"].items():
            assert torch.equal(grads[k], g), (name, k)
        assert torch.equal(x_grad, fx["x_grad"]), name
        torch.manual_seed(fx["sample_seed"])
        assert torch.equal(R.mixture_sample(fx["cls"], fx["state"], 5, fx["x"].shape), fx["sample"]), name


def test_kde_restatement_matches_the_reference(fixture):
    for name, fx in fixture["kde"].items():
        if fx["kernel"] == "GaussianKernel":
            x = fx["x"].clone().requires_grad_(True)
            out = R.gaussian_kde(x, fx["train"], fx["bandwidth"])
            (out * fx["cot"]).sum().backward()
            assert torch.equal(x.grad, fx["x_grad"]), name
        else:
            out = R.parzen_kde(fx["x"], fx["train"], fx["bandwidth"])
        assert torch.equal(out.detach(), fx["out"]), name


def test_float64_restatements_agree_with_the_reference(fixture):
    for name, fx in fixture["mixture"].items():
        out, grads, _ = R.mixture_loss_and_grads(fx["cls"], fx["state"], fx["x"], fx["cot"], torch.float64)
        a, _ = R.mixture_terms(fx["cls"], fx["state"], fx["x"])
        assert torch.allclose(out.float(), fx["out"], rtol=1e-5, atol=1e-4), name
        assert torch.allclose(torch.logsumexp(a, -1).reshape(out.shape), out, rtol=1e-12, atol=1e-10), name
        for k, g in fx["grads"].items():
            assert torch.allclose(grads[k].float(), g, rtol=1e-4, atol=1e-4), (name, k)
    for name, fx in fixture["kde"].items():
        if fx["kernel"] == "GaussianKernel":
            logp, _ = R.gaussian_kde_f64(fx["x"], fx["train"], fx["bandwidth"])
            assert torch.allclose(logp.float(), fx["out"], rtol=1e-5, atol=1e-4), name
        else:
            count = R.parzen_inside(fx["x"], fx["train"], fx["bandwidth"]).sum(1)
            logp = R.parzen_log_density(count, *fx["train"].shape, fx["bandwidth"])
            assert torch.equal(torch.isinf(logp), torch.isinf(fx["out"])), name
            finite = ~torch.isinf(logp)
            assert torch.allclose(logp[finite].float(), fx["out"][finite], rtol=1e-6), name


def test_parzen_boundary_distinguishes_less_or_equal(fixture):
    """The boundary set has queries at fl(|x - t| / h) == 0.5 exactly: the fp32 CPU count with `<` (a bug model)
    differs from the reference, the one with `<=` does not."""
    fx = fixture["kde"]["parzen_boundary"]
    ref = ~torch.isinf(fx["out"])
    good = R.parzen_inside(fx["x"], fx["train"], fx["bandwidth"]).any(1)
    bad = R.parzen_inside(fx["x"], fx["train"], fx["bandwidth"], strict=True).any(1)
    assert torch.equal(good, ref)
    assert not torch.equal(bad, ref)
    q = (fx["x"][:, 0:1] - fx["train"][None, :, 0]).abs() / fx["bandwidth"]
    assert (q == 0.5).any() and (q > 0.5).any() and (q < 0.5).any()


def test_constructor_keys_shapes_order_and_init_bits_match_the_reference(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture["mixture"].items():
        torch.manual_seed(fx["seed"])
        m = getattr(models, fx["cls"])(**fx["kwargs"])
        assert [k for k, _ in m.named_parameters()] == R.mixture_names(fx["cls"]), name
        sd = m.state_dict()
        assert list(sd) == list(fx["state_init"]), name
        for k, v in fx["state_init"].items():
            assert sd[k].dtype == v.dtype and sd[k].shape == v.shape and torch.equal(sd[k], v), (name, k)
        assert (m.n_components, m.n_features) == (fx["kwargs"]["n_components"], fx["kwargs"]["n_features"])
        m.load_state_dict(fx["state"])
    kde = models.KernelDensityEstimator(torch.rand(5, 3))
    assert isinstance(kde.kernel, models.GaussianKernel) and kde.kernel.bandwidth == 1.0
    assert list(kde.state_dict()) == [] and list(kde.parameters()) == [] and "train_Xs" not in dict(kde.named_buffers())
    assert kde.device == torch.device("cpu")
    assert models.ParzenWindowKernel(bandwidth=0.3).bandwidth == 0.3
    with pytest.raises(AssertionError):
        models.KernelDensityEstimator(torch.rand(5, 3, 2))
    with pytest.raises(TypeError):
        models.kde.Kernel()  # abstract, as in the reference


def test_mixture_call_views_the_input_without_shape_buffers():
    from pytorch_generative_b200 import models

    m = models.GaussianMixtureModel(3, 12)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 3, 2, 2))
    assert m._original_shape == (2, 3, 2, 2)
    assert list(m.state_dict()) == ["mixture_logits", "mean", "log_std"]


def test_cpu_and_dtype_refusals():
    from pytorch_generative_b200 import models

    for m in (models.GaussianMixtureModel(3, 4), models.BernoulliMixtureModel(3, 4)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m(torch.zeros(2, 4))
    for kernel in (models.GaussianKernel(), models.ParzenWindowKernel()):
        kde = models.KernelDensityEstimator(torch.rand(5, 3), kernel)
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            kde(torch.rand(2, 3))
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            kernel(torch.rand(2, 3), torch.rand(5, 3))


def test_sample_before_any_forward_raises_attribute_error():
    from pytorch_generative_b200 import models

    for m in (models.GaussianMixtureModel(3, 4), models.BernoulliMixtureModel(3, 4)):
        with pytest.raises(AttributeError):
            m.sample(2)


def test_kde_sample_keeps_the_reference_calls():
    """np.random.choice for the rows, then the kernel's torch noise on the training data's device (CPU here: sampling
    is plain torch)."""
    from pytorch_generative_b200 import models

    train = torch.rand(7, 3)
    for kernel, noise in ((models.GaussianKernel(0.2), lambda s: torch.randn(s) * 0.2),
                          (models.ParzenWindowKernel(0.2), lambda s: (torch.rand(s) - 0.5) * 0.2)):
        kde = models.KernelDensityEstimator(train, kernel)
        np.random.seed(3)
        torch.manual_seed(4)
        got = kde.sample(5)
        np.random.seed(3)
        torch.manual_seed(4)
        idxs = np.random.choice(range(7), size=5)
        assert torch.equal(got, train[idxs] + noise(train[idxs].shape))


def test_gaussian_normaliser_uses_the_reference_fp32_ops():
    from pytorch_generative_b200.models import kde

    for n, d, h in ((100, 2, 1.0), (60000, 784, 0.1), (64, 37, 0.3)):
        nt, ht, pi = torch.tensor(n, dtype=torch.float32), torch.tensor(h), torch.tensor(np.pi)
        ref = 0.5 * d * torch.log(2 * pi) + d * torch.log(ht) + torch.log(nt)
        assert kde.gaussian_log_normaliser(n, d, h) == ref.item()


def test_training_data_that_requires_grad_is_refused():
    """The Gaussian kernel has no gradient with respect to the training data: under autograd recording it raises rather
    than return a gradient that is silently missing (before any device check); without recording it goes on to the
    device check."""
    from pytorch_generative_b200 import models

    t = torch.rand(5, 3, requires_grad=True)
    x = torch.rand(2, 3)
    with pytest.raises(NotImplementedError):
        models.GaussianKernel()(x, t)
    with pytest.raises(NotImplementedError):
        models.KernelDensityEstimator(t)(x)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            models.GaussianKernel()(x, t)


def test_pickle_and_deepcopy():
    from pytorch_generative_b200 import models

    for m in (models.GaussianMixtureModel(3, 4), models.BernoulliMixtureModel(3, 4)):
        for clone in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
            for k, v in m.state_dict().items():
                assert torch.equal(clone.state_dict()[k], v)
    kde = models.KernelDensityEstimator(torch.rand(5, 3), models.ParzenWindowKernel(0.5))
    for clone in (pickle.loads(pickle.dumps(kde)), copy.deepcopy(kde)):
        assert torch.equal(clone.train_Xs, kde.train_Xs) and clone.kernel.bandwidth == 0.5
        assert isinstance(clone.kernel, models.ParzenWindowKernel)


def _stand_in_reference(tmp_path, with_density):
    """A stand-in reference package: the four hot-path models and, when asked for, models/mixture_models.py and
    models/kde.py exporting the five classes from models/__init__.py, as the reference does."""
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
    if with_density:
        (pkg / "models" / "mixture_models.py").write_text(
            "class GaussianMixtureModel:\n    pass\n\nclass BernoulliMixtureModel:\n    pass\n")
        (pkg / "models" / "kde.py").write_text("class KernelDensityEstimator:\n    pass\n\nclass GaussianKernel:\n"
                                               "    pass\n\nclass ParzenWindowKernel:\n    pass\n")
        imports += ("from pytorch_generative.models.mixture_models import BernoulliMixtureModel, GaussianMixtureModel\n"
                    "from pytorch_generative.models.kde import GaussianKernel, KernelDensityEstimator, "
                    "ParzenWindowKernel\n")
    (pkg / "models" / "__init__.py").write_text("from pytorch_generative.models import autoregressive\n" + imports)


DENSITY = {"GaussianMixtureModel": "mixture_models", "BernoulliMixtureModel": "mixture_models",
           "KernelDensityEstimator": "kde", "GaussianKernel": "kde", "ParzenWindowKernel": "kde"}


@pytest.mark.parametrize("with_density", [True, False])
def test_overlay_binds_the_density_models_only_where_the_reference_has_them(tmp_path, with_density):
    _stand_in_reference(tmp_path, with_density)
    sys.path.insert(0, str(tmp_path))
    try:
        import importlib

        import pytorch_generative as ref

        from pytorch_generative_b200 import models, overlay

        orig = {name: getattr(ref.models, name, None) for name in DENSITY}
        bound = overlay.install()
        try:
            assert len(bound) == 14 + 2 * len(DENSITY) * with_density
            for name, mod in DENSITY.items():
                assert (f"pytorch_generative.models.{name}" in bound) == with_density
                assert (f"pytorch_generative.models.{mod}.{name}" in bound) == with_density
                if with_density:
                    assert getattr(ref.models, name) is getattr(models, name)
                    assert getattr(importlib.import_module(f"pytorch_generative.models.{mod}"), name) is \
                        getattr(models, name)
                else:
                    assert not hasattr(ref.models, name)
        finally:
            overlay.uninstall()
        for name in DENSITY:
            assert getattr(ref.models, name, None) is orig[name]
    finally:
        sys.path.remove(str(tmp_path))
        for name in [k for k in sys.modules if k == "pytorch_generative" or k.startswith("pytorch_generative.")]:
            del sys.modules[name]
