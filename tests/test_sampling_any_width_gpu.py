"""Incremental sampling at any channel count: PixelCNN, GatedPixelCNN and PixelSNAIL sample through their per-pixel
programs at widths that are not multiples of 8 (every cache and operand at the padded pitch `round_up(C, 8)`, pad
columns exactly zero), and ImageGPT samples 32 images at widths whose MLP operand no longer fits the skinny GEMM's
shared memory.  Teacher-forced logits against the full forward (two calls: the second replays the captured graph),
the pad columns of every cache, and raster order against the oracle under pre-drawn uniforms.  Tolerances as in
test_parity_gpu.py: 1e-2 of max(1, max|ref|) for the bf16 path."""

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL_BF16 = 1e-2


def dev():
    return torch.device("cuda:0")


def check(name, got, ref, tol):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    bound = tol * max(1.0, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    assert err <= bound and not torch.isnan(got).any(), f"{name}: max err {err:.3e} > {bound:.3e}"


def _pcnn(res, head, c=1):
    return "PixelCNN", dict(in_channels=c, out_channels=c, n_residual=2, residual_channels=res, head_channels=head)


def _gpcnn(gated, head, c=1):
    return "GatedPixelCNN", dict(in_channels=c, out_channels=c, n_gated=2, gated_channels=gated, head_channels=head)


def _snail(ch, key, value, c=1):
    return "PixelSNAIL", dict(in_channels=c, out_channels=c, n_channels=ch, n_pixel_snail_blocks=2, n_residual_blocks=2,
                              attention_key_channels=key, attention_value_channels=value)


# the reference's own multiple-channel smoke configurations (tests/test_channel_counts_gpu.py SMOKE)
SMOKE = [
    ("PixelCNN", dict(in_channels=3, out_channels=3, n_residual=1, residual_channels=1, head_channels=1)),
    ("GatedPixelCNN", dict(in_channels=3, out_channels=3, n_gated=1, gated_channels=1, head_channels=1)),
    ("PixelSNAIL", dict(in_channels=3, out_channels=3, n_channels=2, n_pixel_snail_blocks=1, n_residual_blocks=1,
                        attention_key_channels=1, attention_value_channels=1)),
    ("ImageGPT", dict(in_channels=3, out_channels=3, in_size=8, n_transformer_blocks=1, n_attention_heads=2,
                      n_embedding_channels=4)),
]

SQUARE = (2, 1, 8, 8)
TEACHER_FORCED = (
    [(*_pcnn(r, h), SQUARE) for r in (1, 3, 12) for h in (1, 12)]
    + [(*_gpcnn(g, h), SQUARE) for g in (1, 12, 100) for h in (1, 12)]
    # key / value down to 1, and PixelSNAIL's recipe rule (value = n_channels / 2, key = value / 8)
    + [(*_snail(2, 1, 1), SQUARE), (*_snail(12, 1, 3), SQUARE), (*_snail(12, 1, 6), SQUARE),
       (*_snail(100, 6, 50), SQUARE), (*_snail(100, 1, 1), SQUARE)]
    + [(cls, cfg, (2, 3, 8, 8)) for cls, cfg in SMOKE]
    # non-square images, several image channels
    + [(*_pcnn(3, 5, c=3), (2, 3, 12, 20)), (*_gpcnn(12, 5, c=3), (2, 3, 12, 20)), (*_snail(12, 1, 3, c=3), (2, 3, 12, 20))]
)


def _tol(cls, cfg):
    """TOL_BF16, doubled where a one-ulp difference between the two paths' bf16 operands is amplified: one-channel
    attention keys (the scores are a single product, unaveraged) and LayerNorm over fewer than 8 channels (ImageGPT
    at 4).  Both paths round the same operands to bf16; they differ in summation order only."""
    if cls == "PixelSNAIL" and cfg["attention_key_channels"] == 1:
        return 2 * TOL_BF16
    if cls == "ImageGPT" and cfg["n_embedding_channels"] < 8:
        return 2 * TOL_BF16
    return TOL_BF16


def _ids(cases):
    return [f"{cls}-{'-'.join(str(v) for v in cfg.values())}-{'x'.join(map(str, shape))}" for cls, cfg, shape in cases]


def _pads(cls, m, st):
    """(tensor, true channels, parts) of every padded cache of the per-pixel state: the pad columns of a tensor whose
    `parts` equal parts each hold true channels / parts of them are the columns past each part's true width.  ImageGPT
    keeps no line buffers."""
    if cls == "PixelCNN":
        half = m._input.weight.shape[0] // 2
        return [(st["image"], m._input.weight.shape[1], 1)] + [(t, half, 1) for t in st["t1"]]
    if cls == "GatedPixelCNN":
        C = m._input._out_channels
        return ([(st["image"], st["c"], 1)] + [(t, C, 1) for t in st["vc"] + st["hc"]]
                + [(t, 2 * C, 2) for t in st["v2s"]])
    if cls == "PixelSNAIL":
        C, c = m._input.weight.shape[:2]
        out = [(st["image"], c, 1)]
        for b in st["blocks"]:
            out += [(t, C, 1) for t in b["ea"] + b["eb"]]
            out.append((b["akv"], 2 + C + c, 1))   # [position | features | image | 0-pad]
        return out
    return []


def _check_pads(name, t, channels, parts):
    from pytorch_generative_b200.models import incremental

    width = t.shape[-1]
    part, step = channels // parts, width // parts
    assert width == incremental.pitch(channels, parts), (name, width, channels, parts)
    for g in range(parts):
        pad = t[..., g * step + part: (g + 1) * step]
        assert not pad.any(), f"{name}: pad columns {g * step + part}..{(g + 1) * step} of part {g} are not zero"


def _teacher_forced(m, x, out_channels, tol=TOL_BF16):
    """Per-pixel logits of two teacher-forced calls against the full forward; the per-pixel graph was captured."""
    with torch.no_grad():
        ref = m(x)
    n, c, h, w = x.shape
    assert m._incremental_ok(x)
    for rep in range(2):
        seen = []
        m._sample_fn = lambda logits: (seen.append(logits.detach().clone()), logits.new_zeros(n, c))[1]
        assert torch.equal(m.sample(conditioned_on=x), x)
        assert len(seen) == h * w and all(s.shape == (n, out_channels) for s in seen)
        check(f"incremental logits (call {rep})", torch.stack(seen, dim=-1).view(ref.shape), ref, tol)
    assert m._pixel_states and all(st["graph"] for st in m._pixel_states.values()), "per-pixel program was not graph-captured"


@pytest.mark.parametrize("cls,cfg,shape", TEACHER_FORCED, ids=_ids(TEACHER_FORCED))
def test_incremental_logits_match_the_full_forward_at_any_width(cls, cfg, shape):
    from pytorch_generative_b200 import models

    torch.manual_seed(7)
    m = getattr(models, cls)(**cfg).to(dev())
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.5)
    x = torch.bernoulli(torch.full(shape, 0.5)).to(dev())
    _teacher_forced(m, x, cfg["out_channels"], _tol(cls, cfg))
    for st in m._pixel_states.values():
        for k, (t, channels, parts) in enumerate(_pads(cls, m, st)):
            _check_pads(f"{cls} cache {k}", t, channels, parts)


def test_pad_columns_hold_nonzero_data_beside_them():
    """The pad check above is not vacuous: at 3 residual channels the caches' true columns hold nonzero activations."""
    from pytorch_generative_b200 import models

    torch.manual_seed(3)
    m = models.PixelCNN(**_pcnn(3, 5)[1]).to(dev())
    x = torch.bernoulli(torch.full(SQUARE, 0.5)).to(dev())
    m._sample_fn = lambda logits: logits.new_zeros(SQUARE[0], 1)
    m.sample(conditioned_on=x)
    (st,) = m._pixel_states.values()
    for t in st["t1"]:
        assert t.shape[-1] == 8 and t[..., :3].any() and not t[..., 3:].any()


# --------------------------------------------------------------------------------------------------
# Raster order against the oracle: one odd width per model
# --------------------------------------------------------------------------------------------------
RASTER = {
    "pcnn3": ("pixel_cnn", *_pcnn(3, 5)),
    "gpcnn5": ("gated_pixel_cnn", *_gpcnn(5, 3)),
    "snail6": ("pixel_snail", "PixelSNAIL", dict(in_channels=1, out_channels=1, n_channels=6, n_pixel_snail_blocks=1,
                                                 n_residual_blocks=2, attention_key_channels=1,
                                                 attention_value_channels=3)),
}


@pytest.mark.parametrize("key", sorted(RASTER))
def test_odd_width_sampling_follows_oracle_raster_order(key):
    """Same pre-drawn uniforms in raster order: pixels equal the oracle's sample except, at most, from a knife-edge draw
    (|u - p| within the bf16 tolerance) onwards."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import models

    name, cls, cfg = RASTER[key]
    torch.manual_seed(0)
    m = getattr(models, cls)(**cfg)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=g) * 0.02)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    n, shape = 2, (2, 1, 8, 8)
    u = [torch.rand(n, 1, generator=g) for _ in range(64)]  # one draw per image and pixel, in raster order
    ref = O.sample(name, state, cfg, O.uniform_sample_fn(list(u)), n_samples=n, shape=shape[1:])
    m = m.to(dev())
    m._sample_fn = O.uniform_sample_fn(list(u))
    m(torch.zeros(shape, device=dev()))  # registers the image shape like the reference
    assert m._incremental_ok(torch.zeros(shape, device=dev()))
    got = m.sample(n_samples=n).cpu()
    assert m._pixel_states and all(st["graph"] for st in m._pixel_states.values())
    assert got.shape == ref.shape
    if not torch.equal(got, ref):
        diff = (got != ref).any(dim=1).any(dim=0)
        first = diff.flatten().nonzero()[0].item()
        r, col = divmod(first, shape[3])
        canvas = ref.clone()
        canvas.view(n, 1, -1)[:, :, first:] = -1
        p_ref = torch.sigmoid(O.forward(name, state, canvas, cfg)[:, :, r, col])
        margin = (u[first] - p_ref).abs().min().item()
        assert margin < 2e-2, f"samples diverge at pixel ({r},{col}) without a knife-edge draw (margin {margin:.3e})"


# --------------------------------------------------------------------------------------------------
# Wide ImageGPT: 32 images whose per-pixel MLP operand (32 x 4C bf16) exceeds the skinny GEMM's 160 KiB
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c,heads,blocks", [(648, 6, 2), (1024, 8, 1)])
def test_wide_image_gpt_samples_32_images(c, heads, blocks):
    from pytorch_generative_b200 import models, ops

    assert ops.linear_impl(32, 4 * c, True) != 2  # the contraction this test is about leaves the skinny kernel
    torch.manual_seed(7)
    cfg = dict(in_channels=1, out_channels=1, in_size=8, n_transformer_blocks=blocks, n_attention_heads=heads,
               n_embedding_channels=c)
    m = models.ImageGPT(**cfg).to(dev())
    x = torch.bernoulli(torch.full((32, 1, 8, 8), 0.5)).to(dev())
    _teacher_forced(m, x, 1)
