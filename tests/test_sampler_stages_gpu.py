"""The incremental sampler's per-pixel programs on the H100, stage by stage (tests/_sampler_reference.py,
tests/_sampler_replay.py): every linear, activation, gate, gated residual, LayerNorm, window convolution and KV-cached
attention step of PixelCNN, GatedPixelCNN, PixelSNAIL and ImageGPT against a float64 reference of its recorded inputs
with its per-element bound; every hand-off (operands, residuals, cache rows, the final canvas) bit for bit; the rows
each pixel writes; the logits `sample_fn` receives; every pad column +0.0.  The program runs eagerly for the record
(the capture is made to fail); a second, graph-captured `sample()` under the same uniforms must give the same canvas and
bit-identical logits at every pixel.  A 40 x 32 ImageGPT (1280 keys: the split decode and its merge) is held at the
first and last row and column, and bug models of tests/_sampler_replay.py fail at recipe widths."""

import copy

import pytest
import torch

import _sampler_replay as RP
from test_sampler_bounds_cpu import EMULATED

pytestmark = pytest.mark.gpu

# name -> (model, constructor keywords, canvas shape, partly conditioned, classes of a categorical head)
GEOMETRIES = dict(EMULATED)
GEOMETRIES.update({
    "pixel_cnn-recipe-width": ("pixel_cnn", dict(in_channels=1, out_channels=1, n_residual=3, residual_channels=128,
                                                 head_channels=32), (2, 1, 8, 8), False, None),
    "gated-recipe-width": ("gated_pixel_cnn", dict(in_channels=1, out_channels=1, n_gated=2, gated_channels=128,
                                                   head_channels=32), (2, 1, 8, 8), True, None),
    "snail-recipe-width": ("pixel_snail", dict(in_channels=1, out_channels=1, n_channels=64, n_pixel_snail_blocks=2,
                                               n_residual_blocks=2, attention_key_channels=4,
                                               attention_value_channels=32), (2, 1, 8, 8), False, None),
    # two heads of 64 channels fill their slots; 3 x 256 logits
    "gpt-recipe-width": ("image_gpt", dict(in_channels=3, out_channels=768, in_size=8, n_transformer_blocks=2,
                                           n_attention_heads=2, n_embedding_channels=128), (2, 3, 6, 8), True, 256),
})
CAPTURED = ("pixel_cnn-recipe-width", "gated-recipe-width", "snail-recipe-width", "gpt-recipe-width")
BUG_GEOMETRY = {"pixel_cnn": "pixel_cnn-recipe-width", "snail": "snail-recipe-width"}


def _eager(monkeypatch, geo, m, bug=None, snap=None):
    """The recorded, eager sample() of m on the geometry `geo` (a GEOMETRIES value)."""
    model, kw, shape, cond, classes = geo
    assert m._incremental_ok(torch.zeros(shape, device="cuda")), geo
    if bug is not None:
        RP.BUGS[bug][0](monkeypatch)

    def no_capture(*a, **k):
        raise RuntimeError("capture disabled for the recorded run")
    monkeypatch.setattr(torch.cuda, "CUDAGraph", no_capture)
    with pytest.warns(RuntimeWarning, match="capture"):
        G, rec, out = RP.run(m, model, kw, shape, cond, monkeypatch, classes=classes, snap=snap)
    torch.cuda.synchronize()
    return G, rec, out


@pytest.mark.parametrize("key", list(GEOMETRIES))
def test_every_stage_and_handoff_within_its_bound(key, monkeypatch):
    model, kw = GEOMETRIES[key][:2]
    G, rec, out = _eager(monkeypatch, GEOMETRIES[key], RP.build(model, kw, device="cuda"))
    C = RP.replay(G, rec, out)
    worst = C.worst_by_kind()
    print(f"\n[{key}] worst |err| / bound per check kind")
    print("\n".join(f"  {k:20s} {v:.3e}" for k, v in sorted(worst.items())))
    assert not C.failures, "\n".join(list(C.failures.values())[:10])
    if model in ("pixel_snail", "image_gpt"):
        assert "decode.o" in worst and "handoff.kc" in worst


@pytest.mark.parametrize("key", CAPTURED)
def test_captured_sampler_gives_the_eager_bits(key, monkeypatch):
    """The graph-captured program replayed H x W times gives the eager program's canvas and, at every pixel, its
    logits bit for bit."""
    model, kw, shape, cond, classes = GEOMETRIES[key]
    m = RP.build(model, kw, device="cuda")
    m2 = copy.deepcopy(m)
    fn = m._sample_fn = RP.UniformSampleFn(RP.uniforms(shape, 0), classes)
    with torch.cuda.device(0):
        captured = m.sample(conditioned_on=RP.start_canvas(shape, cond, 0, "cuda"))
    st = next(iter(m._pixel_states.values()))
    assert st["graph"], st.get("graph_error")
    G, rec, eager = _eager(monkeypatch, GEOMETRIES[key], m2)
    assert torch.equal(captured, eager)
    assert len(fn.seen) == len(rec.logits) == shape[2] * shape[3]
    for p, (a, b) in enumerate(zip(fn.seen, rec.logits)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"pixel {p}: logits differ"


def test_split_decode_at_1280_keys(monkeypatch):
    """ImageGPT at 40 x 32: pg_attn_decode splits its 1280 keys over two blocks and merges them.  The decode stage and
    its hand-offs (the K / V rows it reads, its q, k and v) are checked at the first and last row and column."""
    kw = dict(in_channels=1, out_channels=1, in_size=40, n_transformer_blocks=1, n_attention_heads=1,
              n_embedding_channels=16)
    shape = (2, 1, 40, 32)
    h, w = shape[2:]
    edge = {r * w + c for r in range(h) for c in range(w) if r in (0, h - 1) or c in (0, w - 1)}
    G, rec, out = _eager(monkeypatch, ("image_gpt", kw, shape, True, None), RP.build("image_gpt", kw, device="cuda"),
                         snap=edge)
    C = RP.replay(G, rec, out, pixels=edge)
    worst = C.worst_by_kind()
    print("\n".join(f"  {k:20s} {v:.3e}" for k, v in sorted(worst.items())))
    assert not C.failures, "\n".join(list(C.failures.values())[:10])
    assert {"decode.o", "handoff.kc", "handoff.vc"} <= set(worst)


@pytest.mark.parametrize("bug", ["stream_rounded_to_bf16", "decode_not_strict", "kv_fixup_skipped", "taps_wrap_rows"])
def test_bug_model_fails_its_check(bug, monkeypatch):
    key = BUG_GEOMETRY[RP.BUGS[bug][2]]
    model, kw = GEOMETRIES[key][:2]
    G, rec, out = _eager(monkeypatch, GEOMETRIES[key], RP.build(model, kw, device="cuda"), bug)
    failed = RP.replay(G, rec, out).failed_kinds()
    print(f"{bug}: {sorted(failed)}")
    assert RP.BUGS[bug][1] in failed, (bug, sorted(failed))
