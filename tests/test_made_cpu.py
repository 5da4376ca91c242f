"""MADE without a GPU: the CPU restatement (tests/_made_reference.py) against the reference's own outputs
(tests/golden/made.pt), the model's constructor, state-dict keys, connectivity vectors and mask rotation, the refusal to
run on CPU tensors, and the recipe's signature."""

import inspect
import os

import numpy as np
import pytest
import torch

import _made_reference as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "made.pt")


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _close(a, b, tol=1e-5):
    return (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())


def test_reference_restatement_matches_the_reference(fixture):
    for name, fx in fixture.items():
        n_masks = fx["kwargs"].get("n_masks", 1)
        p = {k: v.clone() for k, v in fx["state_before"].items()}
        for f, step in enumerate(fx["forwards"]):
            logits, loss, grads, x_grad, p = R.loss_and_grads(p, step["x"], f, n_masks)
            assert _close(logits, step["logits"]), name
            assert _close(loss, step["loss"]), name
            assert _close(x_grad, step["x_grad"]), name
            for k, g in step["grads"].items():
                assert _close(grads[k], g), (name, k)
            for k, m in step["masks"].items():
                assert torch.equal(p[k], m.float()), (name, k)
        for k in fx["state_before"]:  # masked weights and the last mask set (state_after adds _c/_h/_w)
            assert torch.equal(p[k], fx["state_after"][k]), (name, k)
        for kind in ("unconditional", "conditional"):
            s = fx[kind]
            start = s["conditioned_on"] if s["conditioned_on"] is not None else -torch.ones_like(s["sample"])
            got = R.sample(fx["state_after"], s["mask_seed_before"], R.uniform_sample_fn(s["uniforms"]), start, n_masks)
            assert torch.equal(got, s["sample"]), (name, kind)


def test_constructor_and_state_dict_keys_match_the_reference(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture.items():
        m = models.MADE(**fx["kwargs"])
        sd = m.state_dict()
        assert set(sd) == set(fx["state_before"]), name
        for k, v in fx["state_before"].items():
            assert sd[k].shape == v.shape and sd[k].dtype == v.dtype, (name, k)
        m.load_state_dict(fx["state_after"])  # including the _c/_h/_w buffers of an image forward
        assert int(m._c) * int(m._h) * int(m._w) == fx["kwargs"]["input_dim"]
    sig = inspect.signature(models.MADE.__init__)
    assert [(k, v.default) for k, v in sig.parameters.items()][1:] == [
        ("input_dim", inspect.Parameter.empty), ("hidden_dims", None), ("n_masks", 1), ("sample_fn", None)]
    from pytorch_generative_b200.models.made import MaskedLinear

    lin = MaskedLinear(5, 3)
    assert set(lin.state_dict()) == {"weight", "bias", "mask"} and torch.equal(lin.mask, torch.ones(3, 5))
    lin.set_mask(torch.zeros(3, 5, dtype=torch.uint8))
    assert not lin.mask.any()
    assert list(inspect.signature(MaskedLinear.__init__).parameters) == ["self", "in_features", "out_features", "bias"]


def test_connectivity_and_masks_equal_the_reference(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture.items():
        m = models.MADE(**fx["kwargs"])
        hidden = fx["kwargs"].get("hidden_dims") or []
        assert fx["connectivity"], name
        for mask_set, recorded in fx["connectivity"].items():
            vecs = m._connectivity(mask_set)
            assert len(vecs) == len(hidden) + 2
            for got, want in zip(vecs, recorded):  # the reference's permutation and randint draws
                assert np.array_equal(got, want.numpy()), (name, mask_set)
            assert np.array_equal(vecs[-1], vecs[0])
            assert np.array_equal(vecs[0], R.connectivity(fx["kwargs"]["input_dim"], hidden, mask_set)[0])
        n_masks = fx["kwargs"].get("n_masks", 1)
        for f, step in enumerate(fx["forwards"]):
            built = R.masks(m._connectivity(f % n_masks))
            for layer, mask in enumerate(built):
                assert torch.equal(mask, step["masks"][f"_net.{2 * layer}.mask"].float()), (name, f, layer)


def test_mask_seed_advances_like_the_reference(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture.items():
        m = models.MADE(**fx["kwargs"])
        n_masks = fx["kwargs"].get("n_masks", 1)
        sets = [m._next_mask_set() for _ in fx["forwards"]]  # one per forward
        assert sets == [f % n_masks for f in range(len(fx["forwards"]))]
        for kind in ("unconditional", "conditional"):  # one per sample call
            assert m._mask_seed == fx[kind]["mask_seed_before"], (name, kind)
            m._next_mask_set()
        assert m._mask_seed == fx["mask_seed_after"], name


def test_forward_and_sample_refuse_cpu_tensors():
    from pytorch_generative_b200 import models
    from pytorch_generative_b200.models.made import MaskedLinear

    m = models.MADE(16, [8])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 16))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.sample(conditioned_on=-torch.ones(2, 16))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        MaskedLinear(4, 4)(torch.zeros(1, 4))


def test_reproduce_made_signature():
    from pytorch_generative_b200 import recipes
    from pytorch_generative_b200.models import made

    sig = inspect.signature(recipes.reproduce_made)
    assert {k: v.default for k, v in sig.parameters.items()} == dict(
        n_epochs=85, batch_size=64, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None)
    assert made.reproduce.__doc__ and "reproduce_made" in inspect.getsource(made.reproduce)
    with pytest.raises(RuntimeError, match="CUDA"):
        recipes.reproduce_made(n_gpus=0, debug_loader=[])
