"""ImageGPT's fused stack on the H100, stage by stage (tests/_block_reference.py): every activation the forward saves,
every gradient the backward hands between its kernels and every parameter gradient, each against a float64 reference
computed from that stage's own inputs chosen by role (parameters, cotangent, saved activations, recorded
intermediates), with the per-element bound of the stage's kernel; every pad column and every pad row of the packed
gradients exactly zero.  Then a second identical step gives identical bits, and the bug models of
tests/_block_replay.py that change only which valid tensor or argument the product passes fail at real sizes.

Parameters sit well away from their initialisation (LayerNorm gammas 1 + 0.5 N(0, 1), nonzero betas, biases and
positional parameter) and the cotangent is unit-scale.  The store path is forced: the recompute path is held
bit-identical to it elsewhere (test_channel_counts_gpu.py, test_imagegpt_recompute_gpu.py)."""

import pytest
import torch

import _block_replay as RP

pytestmark = pytest.mark.gpu

# name -> (channels, heads, images n x cin x h x w); out_channels = cin
GEOMETRIES = {
    "C512-8heads-2x3x32x32": (512, 8, (2, 3, 32, 32)),    # the C5 recipe: heads fill their slots, arena packing
    "C512-4heads-2x3x32x32": (512, 4, (2, 3, 32, 32)),    # dk = 128
    "C64-4heads-2x1x28x28": (64, 4, (2, 1, 28, 28)),      # the C2 width: dk 16 in 64-wide slots, S = 784
    "C100-4heads-2x3x12x20": (100, 4, (2, 3, 12, 20)),    # padded stream (c_p 104, f_p 400), dk 25
    "C12-3heads-3x1x7x9": (12, 3, (3, 1, 7, 9)),
    "C256-2heads-1x3x48x48": (256, 2, (1, 3, 48, 48)),    # S = 2304: many key tiles, the last one ragged
}
SENSITIVITY = ["C512-8heads-2x3x32x32", "C100-4heads-2x3x12x20"]


def _store_path(monkeypatch):
    from pytorch_generative_b200.models import image_gpt

    monkeypatch.setattr(image_gpt.ImageGPT, "_recompute_for", lambda self, x: False)


def _run(monkeypatch, key, bug=None):
    C, heads, shape = GEOMETRIES[key]
    _store_path(monkeypatch)
    m, x, G = RP.build(C, heads, shape, cout=shape[1], device="cuda")
    if bug is not None:
        RP.BUGS[bug][0](monkeypatch)
    rec = RP.Recorder(monkeypatch)
    logits, sv, blocks = RP.step(m, x, G, rec, lambda model, inp: model(inp))
    return m, x, G, logits, RP.replay(m, x, G, logits, sv, blocks, rec), rec


@pytest.mark.parametrize("key", list(GEOMETRIES))
def test_every_stage_within_its_bound(key, monkeypatch):
    m, x, G, logits, mode, rec = _run(monkeypatch, key)
    worst = mode.worst_by_kind()
    print(f"\n[{key}] worst |err| / bound per stage")
    print("\n".join(f"  {k:28s} {v:.3e}" for k, v in sorted(worst.items())))
    assert not mode.failures, "\n".join(mode.failures.values())
    assert sum(k.startswith("grad ") for k in worst) == 21 and len(rec.arena) == 2

    # a second identical step: the same bits for the logits and every gradient
    first = {n: p.grad.clone() for n, p in m.named_parameters()}
    logits2, _, _ = RP.step(m, x, G, rec, lambda model, inp: model(inp))
    assert torch.equal(logits2, logits)
    for n, p in m.named_parameters():
        assert torch.equal(p.grad, first[n]), f"second step: {n}"


@pytest.mark.parametrize("bug", sorted(RP.BUGS))
@pytest.mark.parametrize("key", SENSITIVITY)
def test_bug_model_fails_at_real_size(key, bug, monkeypatch):
    from pytorch_generative_b200.nn.modules import head_layout

    C, heads, _ = GEOMETRIES[key]
    apply, stage, narrow_heads_only = RP.BUGS[bug]
    if narrow_heads_only and head_layout(heads, C, C).identity:
        pytest.skip("heads fill their slots: no scatter packing, and the slot width is the head width")
    *_, mode, _ = _run(monkeypatch, key, bug)
    failed = mode.failed_kinds()
    print(f"\n[{key}] {bug}: fails {failed}")
    assert stage in failed, (bug, failed)
