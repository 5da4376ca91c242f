"""The bf16 weight copies under CUDA-graph replay and in eval: a replayed training step must invalidate the copies an
eager forward made before it, a refresh captured in the step must keep writing the step's own arena whatever eager
refreshes run between replays, and unchanged weights must not be cast again."""

import re

import pytest
import torch

pytestmark = pytest.mark.gpu

IGPT_IDENTITY = ("ImageGPT", dict(in_channels=1, out_channels=1, in_size=8, n_transformer_blocks=2, n_attention_heads=2,
                                  n_embedding_channels=128), (2, 1, 8, 8))
MODELS = {
    "image_gpt_identity": IGPT_IDENTITY,
    "image_gpt_padded": ("ImageGPT", dict(in_channels=1, out_channels=1, in_size=8, n_transformer_blocks=2,
                                          n_attention_heads=4, n_embedding_channels=64), (2, 1, 8, 8)),
    "gated_pixel_cnn": ("GatedPixelCNN", dict(in_channels=3, out_channels=3, n_gated=2, gated_channels=64,
                                              head_channels=32), (2, 3, 8, 16)),
    "pixel_snail": ("PixelSNAIL", dict(in_channels=3, out_channels=3, n_channels=64, n_pixel_snail_blocks=2,
                                       n_residual_blocks=2, attention_key_channels=16, attention_value_channels=32),
                    (2, 3, 16, 16)),
}


def dev():
    return torch.device("cuda:0")


def _model(cls, cfg, seed=0):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    return getattr(models, cls)(**cfg).to(dev()).train()


def _batches(shape, n, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [torch.bernoulli(torch.full(shape, 0.5), generator=g).to(dev()) for _ in range(n)]


def _graphed(m, x):
    from pytorch_generative_b200 import losses, trainstep

    return trainstep.GraphedTrainStep(m, list(m.parameters()), lambda p, t: losses.bce_with_logits_sum_mean(p, t), x,
                                      lr=5e-3, lr_gamma=0.999977)


@pytest.mark.parametrize("name", sorted(MODELS))
def test_eager_forward_after_a_replay_reads_the_replayed_weights(name):
    """replay, eager forward, replay, eager forward: the last forward computes with the weights of the second replay,
    exactly as a fresh model loaded with them does."""
    cls, cfg, shape = MODELS[name]
    m = _model(cls, cfg)
    xs = _batches(shape, 3)
    step = _graphed(m, xs[0])
    step(xs[1])
    with torch.no_grad():
        m(xs[0])  # makes copies of the weights of the first replay
    step(xs[2])
    with torch.no_grad():
        got = m(xs[0])
    fresh = _model(cls, cfg, seed=1)
    fresh.load_state_dict(m.state_dict())
    with torch.no_grad():
        want = fresh(xs[0])
    assert torch.equal(got, want)


def test_eager_refreshes_between_replays_leave_the_training_step_unchanged():
    """ImageGPT with heads that fill their slots (one-cast arena): three replays with an eager forward and a sample()
    between them train exactly like three replays alone."""
    cls, cfg, shape = IGPT_IDENTITY
    xs = _batches(shape, 3)
    runs = []
    for interleave in (False, True):
        m = _model(cls, cfg)
        m._sample_fn = lambda logits: (logits > 0).float()  # no random draws: the two runs differ only by the refreshes
        step = _graphed(m, xs[0])
        step.reset({k: v.clone() for k, v in _model(cls, cfg).state_dict().items()})
        out = []
        for i, x in enumerate(xs):
            out.append(step(x))
            if interleave and i < len(xs) - 1:
                with torch.no_grad():
                    m(x[:1])
                m.sample(n_samples=2)
        runs.append((out, [p.detach().clone() for p in m.parameters()]))
    (out_a, params_a), (out_b, params_b) = runs
    assert out_a == out_b
    for a, b in zip(params_a, params_b):
        assert torch.equal(a, b)


def _cast_launches(fn):
    """Number of pg_cast_f32_to_bf16 kernels (`cast_kernel`) that fn() launches."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, sum(e.count for e in prof.key_averages() if re.search(r"(?<![A-Za-z_])cast_kernel", e.key))


def test_unchanged_weights_are_not_cast_again():
    """Two eval forwards of PixelSNAIL: the first casts its convolution and attention weights, the second reuses them
    and computes the same logits."""
    cls, cfg, shape = MODELS["pixel_snail"]
    m = _model(cls, cfg).eval()
    (x,) = _batches(shape, 1)
    with torch.no_grad():
        first, n_first = _cast_launches(lambda: m(x))
        second, n_second = _cast_launches(lambda: m(x))
    assert n_first > 0
    assert n_second == 0
    assert torch.equal(first, second)
