"""The incremental sampler's per-pixel programs stage by stage, without a GPU (tests/_sampler_reference.py,
tests/_sampler_emulation.py, tests/_sampler_replay.py).

1. The stage references, chained in float64 along the stage graph at every pixel of a canvas, reproduce the logits of
   oracle/reference_path.py's full forward to 1e-10 relative.  This holds the graph (tap offsets, paddings, caches,
   fix-ups, layouts) to the reference independently of the product.
2. The product's own `sample()` runs its programs on fp32 CPU stand-ins of the kernels, and every stage value, hand-off,
   cache row and pad column passes the checks the GPU test holds the kernels to, for unconditional and partly
   conditioned canvases.  The geometries reach channel counts that are not multiples of 8 in every model, GatedPixelCNN
   with two gated layers, PixelSNAIL with two blocks and key width 3, ImageGPT heads in padded and in filled slots,
   non-square images and a 256 x 2-way categorical head.
3. Each bug model (tests/_sampler_replay.BUGS), applied alone, fails the check it names."""

import pytest
import torch

import _sampler_emulation as E
import _sampler_reference as R
import _sampler_replay as RP
from oracle import reference_path as O

F64 = torch.float64

_PCNN = dict(in_channels=1, out_channels=1, n_residual=2, residual_channels=6, head_channels=5)
_GATED = dict(in_channels=1, out_channels=1, n_gated=2, gated_channels=10, head_channels=6)
_SNAIL = dict(in_channels=1, out_channels=1, n_channels=12, n_pixel_snail_blocks=2, n_residual_blocks=1,
              attention_key_channels=3, attention_value_channels=6)
_GPT = dict(in_channels=1, out_channels=1, in_size=6, n_transformer_blocks=2, n_attention_heads=2,
            n_embedding_channels=12)
# name -> (model, constructor keywords, canvas shape, partly conditioned, classes of a categorical head)
EMULATED = {
    "pixel_cnn": ("pixel_cnn", _PCNN, (2, 1, 5, 7), False, None),
    "pixel_cnn-cond": ("pixel_cnn", _PCNN, (2, 1, 5, 7), True, None),
    "gated": ("gated_pixel_cnn", _GATED, (2, 1, 6, 5), False, None),
    "gated-cond": ("gated_pixel_cnn", _GATED, (2, 1, 6, 5), True, None),
    "snail": ("pixel_snail", _SNAIL, (2, 1, 5, 6), False, None),
    "snail-cond": ("pixel_snail", _SNAIL, (2, 1, 5, 6), True, None),
    # two heads of 6 channels, each in a 64-wide slot
    "gpt": ("image_gpt", _GPT, (2, 1, 5, 6), False, None),
    "gpt-cond": ("image_gpt", _GPT, (2, 1, 5, 6), True, None),
    # one head of 64 channels: the slot is filled and the packing is the identity
    "gpt-filled": ("image_gpt", dict(in_channels=1, out_channels=1, in_size=4, n_transformer_blocks=1,
                                     n_attention_heads=1, n_embedding_channels=64), (2, 1, 4, 4), True, None),
    # 2 image channels, 256 classes each: 512 logits per pixel, class k of channel c at 2 k + c
    "categorical": ("pixel_cnn", dict(in_channels=2, out_channels=512, n_residual=1, residual_channels=4,
                                      head_channels=12), (2, 2, 4, 4), True, 256),
}
BUG_GEOMETRY = {"pixel_cnn": "pixel_cnn", "gated": "gated", "snail": "snail", "gpt": "gpt",
                "categorical": "categorical"}


@pytest.mark.parametrize("geo", sorted(EMULATED))
def test_stage_chain_matches_the_oracle(geo):
    model, kw, shape, _, classes = EMULATED[geo]
    m = RP.build(model, kw)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    canvas = torch.randint(0, classes or 2, shape, generator=g).to(F64) / ((classes or 2) - 1)
    got = R.chain(R.graph(model, state, shape, kw.get("n_attention_heads")), canvas)
    P = {k: v.to(F64).clone() for k, v in state.items()}
    if model == "image_gpt":
        P["_pos"] = P["_pos"][:, :, : shape[2], : shape[3]]
    ref = O.forward(model, P, canvas, dict(n_attention_heads=kw.get("n_attention_heads")))
    assert float((got - ref).abs().max() / ref.abs().max()) <= 1e-10


def _emulated(monkeypatch, geo, bug=None):
    E.install(monkeypatch)
    model, kw, shape, cond, classes = EMULATED[geo]
    m = RP.build(model, kw)
    assert m._incremental_ok(torch.zeros(shape)), geo  # else sample() would fall back and check nothing
    if bug is not None:
        RP.BUGS[bug][0](monkeypatch)
    with pytest.warns(RuntimeWarning, match="capture"):
        G, rec, out = RP.run(m, model, kw, shape, cond, monkeypatch, classes=classes)
    return G, RP.replay(G, rec, out), out


@pytest.mark.parametrize("geo", sorted(EMULATED))
def test_emulated_sampler_passes_every_check(geo, monkeypatch):
    G, C, out = _emulated(monkeypatch, geo)
    print("\n".join(f"{k:24s} {v:.3e}" for k, v in sorted(C.worst_by_kind().items())))
    assert not C.failures, "\n".join(list(C.failures.values())[:10])
    assert (out >= 0).all()
    kinds = C.worst_by_kind()
    for kind in ("handoff.a", "linear.y", "cache.final", "logits.order"):
        assert kind in kinds, sorted(kinds)
    if EMULATED[geo][0] in ("pixel_snail", "image_gpt"):
        assert "decode.o" in kinds and "handoff.kc" in kinds


@pytest.mark.parametrize("bug", sorted(RP.BUGS))
def test_bug_model_fails_its_check(bug, monkeypatch):
    _, C, _ = _emulated(monkeypatch, BUG_GEOMETRY[RP.BUGS[bug][2]], bug)
    failed = C.failed_kinds()
    print(f"{bug}: {sorted(failed)}")
    assert RP.BUGS[bug][1] in failed, (bug, sorted(failed))
