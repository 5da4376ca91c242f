"""Host-side logic that needs no GPU: trainer checkpoint plumbing, FusedAdam's chunk plan, data transforms, recipe
signatures (reference trainer.py:98-148, datasets.py:16-25, the `reproduce` signatures of the four recipes)."""

import inspect

import pytest
import torch


def test_strip_ddp_prefix():
    from pytorch_generative_b200 import trainer

    sd = {"module._input.weight": torch.zeros(1), "module._c": torch.tensor(1)}
    assert list(trainer.strip_ddp_prefix(sd)) == ["_input.weight", "_c"]
    plain = {"_input.weight": torch.zeros(1)}
    assert trainer.strip_ddp_prefix(plain) is plain


def test_trainer_constructor_matches_reference_signature():
    from pytorch_generative_b200 import trainer

    params = list(inspect.signature(trainer.Trainer.__init__).parameters)
    assert params == ["self", "model", "loss_fn", "optimizer", "train_loader", "eval_loader", "lr_scheduler",
                      "clip_grad_norm", "skip_grad_norm", "log_dir", "sample_epochs", "save_checkpoint_epochs", "n_gpus",
                      "device_id"]
    for name in ("interleaved_train_and_eval", "restore_checkpoint", "train_one_batch", "eval_one_batch", "sample_one_batch",
                 "_train_one_batch", "_eval_one_batch", "_save_checkpoint"):
        assert hasattr(trainer.Trainer, name)


@pytest.mark.parametrize("mod,batch", [("pixel_cnn", 256), ("gated_pixel_cnn", 128), ("pixel_snail", 128), ("image_gpt", 64)])
def test_reproduce_signatures(mod, batch):
    """`reproduce(n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)` with the reference defaults; the CUDA
    path refuses n_gpus=0 instead of falling back to the CPU."""
    import importlib

    m = importlib.import_module(f"pytorch_generative_b200.models.{mod}")
    from pytorch_generative_b200 import recipes

    fn = getattr(recipes, f"reproduce_{mod}")
    sig = inspect.signature(fn)
    assert list(sig.parameters) == ["n_epochs", "batch_size", "log_dir", "n_gpus", "device_id", "debug_loader"]
    assert sig.parameters["n_epochs"].default == 457 and sig.parameters["batch_size"].default == batch
    assert sig.parameters["log_dir"].default == "/tmp/run" and sig.parameters["n_gpus"].default == 1
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.reproduce(n_epochs=1, batch_size=2, n_gpus=0, debug_loader=[torch.zeros(2, 1, 28, 28)])


def test_fused_adam_plan_and_state_layout():
    from pytorch_generative_b200 import optim

    ps = [torch.zeros(3), torch.zeros(5, 5)]
    opt = optim.FusedAdam(ps, lr=1e-3)
    ref = torch.optim.Adam([torch.zeros(3), torch.zeros(5, 5)], lr=1e-3)
    assert set(opt.param_groups[0]) >= {"lr", "betas", "eps", "weight_decay", "amsgrad"}
    assert opt.param_groups[0]["betas"] == ref.param_groups[0]["betas"] and opt.param_groups[0]["eps"] == ref.param_groups[0]["eps"]
    ps[0].grad = torch.ones(3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        opt.step()
    with pytest.raises(NotImplementedError):
        optim.FusedAdam(ps, weight_decay=0.1)


def test_device_transforms_on_cpu():
    from pytorch_generative_b200 import datasets

    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (4, 1, 28, 28), dtype=torch.uint8, generator=g)
    loader = [(x, torch.zeros(4, dtype=torch.long))]
    (xb, yb), = list(datasets.DeviceTransform(loader, "cpu", binarize=True, seed=1))
    assert xb.dtype == torch.float32 and set(xb.unique().tolist()) <= {0.0, 1.0} and yb.shape == (4,)
    (xd,), = [b[:1] for b in datasets.DeviceTransform(loader, "cpu", dequant=True, pad_to_32=True, seed=1)]
    assert xd.shape == (4, 1, 32, 32) and float(xd.max()) < 1.0 and float(xd[:, :, 2:-2, 2:-2].min()) >= 0.0
    with pytest.raises(ValueError):
        datasets.DeviceTransform(loader, "cpu", binarize=True, dequant=True)
    # dynamic binarisation keeps the pixel mean (Bernoulli(p = pixel))
    big = torch.full((1, 1, 256, 256), 0.3)
    assert abs(datasets.dynamically_binarize(big, g).mean().item() - 0.3) < 0.01


def test_models_copy_and_pickle_without_their_pixel_states_and_cast_plan():
    """sample() / training leave per-instance caches (captured CUDA graphs, line buffers, ImageGPT's cast plan) in the
    module's __dict__; copy.deepcopy / pickle must drop them instead of failing on (or sharing) them.  The bf16 weight
    copies are not on the module: test_weight_cache_cpu checks that a deep copy's Parameters find none of them."""
    import copy
    import pickle
    import threading

    from pytorch_generative_b200 import models

    m = models.PixelCNN(in_channels=1, out_channels=1, n_residual=1, residual_channels=8, head_channels=8)
    unpicklable = threading.Lock()  # stands for a torch.cuda.CUDAGraph
    m.__dict__["_pixel_states"] = {("key",): dict(graph=unpicklable)}
    c = copy.deepcopy(m)
    assert "_pixel_states" not in c.__dict__
    assert "_pixel_states" in m.__dict__  # the original keeps its caches
    for (k, a), (_, b) in zip(m.state_dict().items(), c.state_dict().items()):
        assert torch.equal(a, b), k
    r = pickle.loads(pickle.dumps(m))
    assert "_pixel_states" not in r.__dict__ and set(r.state_dict()) == set(m.state_dict())
    g = models.ImageGPT(in_channels=1, out_channels=1, in_size=4, n_transformer_blocks=1, n_attention_heads=1,
                        n_embedding_channels=8)
    g.__dict__["_pixel_states"] = {("key",): dict(graph=unpicklable)}
    g.__dict__["_cast_plan"] = dict(src_key=None, src=unpicklable)
    c = copy.deepcopy(g)
    assert "_pixel_states" not in c.__dict__ and "_cast_plan" not in c.__dict__
    assert "_pixel_states" in g.__dict__ and "_cast_plan" in g.__dict__
