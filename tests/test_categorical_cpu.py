"""CPU checks of the categorical likelihood: the float64 restatement against F.cross_entropy, the target rule on the 8-bit
grid, the bits/dim arithmetic and argument checks of losses.categorical_nll, the sample function's signature and
pickling, the 8-bit recipe's signature and the library's new symbols."""

import copy
import inspect
import math
import pickle

import pytest
import torch
import torch.nn.functional as F

import _categorical_reference as R

F64 = torch.float64


@pytest.mark.parametrize("K", [2, 17, 256])
@pytest.mark.parametrize("C", [1, 3, 4])
def test_restatement_matches_cross_entropy(K, C):
    g = torch.Generator().manual_seed(K * 10 + C)
    N, H, W = 3, 5, 7
    logits = (torch.randn(N, K * C, H, W, generator=g) * 3).float()
    x = torch.randint(0, K, (N, C, H, W), generator=g).float() / (K - 1)
    t = R.target(x, K)
    want = F.cross_entropy(logits.to(F64).reshape(N, K, C, H, W), t, reduction="none")
    assert (R.nll(logits, x) - want).abs().max().item() <= 1e-12
    loss, bpd = R.loss(logits, x)
    assert abs(loss.item() - want.sum(dim=(1, 2, 3)).mean().item()) <= 1e-12 * max(1.0, loss.item())
    assert abs(bpd.item() - loss.item() / (C * H * W * math.log(2))) <= 1e-12
    lv = logits.to(F64).requires_grad_(True)
    F.cross_entropy(lv.reshape(N, K, C, H, W), t, reduction="sum").mul(0.25).backward()
    assert (R.dlogits(logits, x, 0.25) - lv.grad).abs().max().item() <= 1e-12


@pytest.mark.parametrize("K", [2, 17, 256])
def test_target_rule_is_exact_on_the_grid(K):
    """x = k / (K - 1) in fp32 (what the loaders produce for K = 256) gives class k for every k, in the product's rule
    and the restatement's; values outside [0, 1] clamp to the end classes."""
    from pytorch_generative_b200 import losses

    k = torch.arange(K)
    x = k.float() / (K - 1)
    assert torch.equal(losses.categorical_target(x, K), k)
    assert torch.equal(R.target(x, K), k)
    if K == 256:  # the loaders' uint8 / 255
        assert torch.equal(losses.categorical_target(k.to(torch.uint8).float() / 255, K), k)
    ends = torch.tensor([-0.5, -0.0, 1.0, 1.5, float("inf"), -float("inf")])
    assert losses.categorical_target(ends, K).tolist() == [0, 0, K - 1, K - 1, K - 1, 0]


def test_bits_per_dim_arithmetic(monkeypatch):
    """categorical_nll divides its loss by C H W ln 2 (the autograd Function is replaced by the restatement so the
    arithmetic runs on the CPU)."""
    from pytorch_generative_b200 import losses

    monkeypatch.setattr(losses._CategoricalNLL, "apply", lambda p, x: R.loss(p, x)[0])
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(2, 256 * 3, 4, 6, generator=g)
    x = torch.randint(0, 256, (2, 3, 4, 6), generator=g).float() / 255
    out = losses.categorical_nll(x, None, logits)
    assert set(out) == {"loss", "bits_per_dim"}
    ref, ref_bpd = R.loss(logits, x)
    assert out["loss"].item() == ref.item()
    assert abs(out["bits_per_dim"].item() - ref.item() / (3 * 4 * 6 * math.log(2))) <= 1e-12 * ref_bpd.item()
    assert abs(out["bits_per_dim"].item() - ref_bpd.item()) <= 1e-12 * ref_bpd.item()


@pytest.mark.parametrize("preds_shape,x_shape", [
    ((2, 10, 4, 4), (2, 3, 4, 4)),     # 10 logit channels are not K * 3
    ((2, 3, 4, 4), (2, 3, 4, 4)),      # K = 1
    ((2, 768, 4, 4), (2, 3, 4, 5)),    # spatial shapes differ
    ((3, 768, 4, 4), (2, 3, 4, 4)),    # batch sizes differ
    ((2, 768, 16), (2, 3, 4, 4)),      # ranks differ
])
def test_argument_checks(preds_shape, x_shape):
    from pytorch_generative_b200 import losses

    with pytest.raises(ValueError):
        losses.categorical_nll(torch.zeros(x_shape), None, torch.zeros(preds_shape))


def test_no_cpu_fallback():
    from pytorch_generative_b200 import losses, models

    with pytest.raises(RuntimeError):
        losses.categorical_nll(torch.zeros(1, 1, 2, 2), None, torch.zeros(1, 256, 2, 2))
    with pytest.raises(RuntimeError):
        models.categorical_sample_fn()(torch.zeros(2, 256))


def test_sample_fn_signature_and_pickling():
    from pytorch_generative_b200 import models

    sig = inspect.signature(models.categorical_sample_fn)
    assert list(sig.parameters) == ["n_classes"] and sig.parameters["n_classes"].default == 256
    fn = models.categorical_sample_fn(17)
    assert isinstance(fn, models.CategoricalSampleFn) and fn.n_classes == 17
    for twin in (pickle.loads(pickle.dumps(fn)), copy.deepcopy(fn)):
        assert type(twin) is models.CategoricalSampleFn and twin.n_classes == 17
    with pytest.raises(ValueError):
        models.categorical_sample_fn(1)
    with pytest.raises(ValueError):
        fn(torch.zeros(2, 18))  # not a multiple of 17 classes
    # a model that carries it pickles and deep-copies like any other
    m = models.PixelCNN(in_channels=1, out_channels=256, n_residual=1, residual_channels=8, head_channels=8,
                        sample_fn=models.categorical_sample_fn())
    for twin in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
        assert twin._sample_fn.n_classes == 256


def test_recipe_signature():
    from pytorch_generative_b200 import recipes

    sig = inspect.signature(recipes.reproduce_image_gpt_8bit)
    ref = inspect.signature(recipes.reproduce_image_gpt)
    assert list(sig.parameters) == list(ref.parameters)
    assert {k: p.default for k, p in sig.parameters.items()} == {k: p.default for k, p in ref.parameters.items()}
    assert "not validated" in recipes.reproduce_image_gpt_8bit.__doc__


def test_build_exports_the_new_symbols():
    from pytorch_generative_b200 import _build, _lib

    _build.build(verbose=False)
    lib = _lib.load()
    for sym in ("pg_categorical_xent_fwd_bwd", "pg_categorical_sample"):
        assert sym in _lib.EXPORTED_SYMBOLS
        getattr(lib, sym)
