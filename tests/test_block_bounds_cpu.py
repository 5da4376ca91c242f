"""ImageGPT's fused stack stage by stage, without a GPU (tests/_block_reference.py, tests/_block_replay.py).

1. The stage references, chained in float64 on their own outputs, are the oracle's model: logits and the gradient of
   every parameter equal oracle/reference_path.py's image_gpt_forward and its autograd to 1e-10 relative (head split,
   double residual, attention scale, which column sums feed which bias).
2. The product's own wiring (`_ImageGPTStack`, `_block_fwd`, `_block_bwd`, `GradArena`, the weight packing) runs on
   fp32 CPU stand-ins of the kernels (tests/_block_emulation.py), and every stage, parameter gradient and pad passes
   the bounds the GPU test holds the kernels to.  Heads narrower than their slots take the general packing branch; the
   slot-filling branch packs through device pointer tables and is covered on the GPU only.
3. Each bug model (tests/_block_replay.BUGS), applied alone to the emulated stack, fails the stage it names."""

import pytest
import torch

import _block_emulation as E
import _block_reference as R
import _block_replay as RP

F64 = torch.float64


@pytest.mark.parametrize("C,heads", [(12, 3), (128, 2)], ids=["padded-heads", "slot-filling"])
def test_stage_chain_matches_the_oracle(C, heads):
    from oracle import reference_path as O

    m, x, G = RP.build(C, heads, (2, 2, 6, 6), cout=3)
    pt = O.trainable({k: v.detach().to(F64) for k, v in m.state_dict().items()})
    x64, G64 = x.to(F64), G.to(F64)
    ref_logits = O.image_gpt_forward(pt, x64, heads)
    (ref_logits * G64).sum().backward()

    g = RP.geometry(m, x)
    chain = R.Chain()
    W = R.weights(pt, len(m._transformer), lambda t: t)
    logits = R.run(W, g, x64 + pt["_pos"].detach(), G64.permute(0, 2, 3, 1).reshape(g.P, g.cout), m._ln.eps, chain)

    def rel(got, ref):
        return float((got - ref).abs().max() / ref.abs().max())

    assert rel(logits, ref_logits.detach().permute(0, 2, 3, 1).reshape(g.P, g.cout)) <= 1e-10
    expected = {k for k, v in pt.items() if v.grad is not None}
    assert set(chain.grads) == expected == {k for k, _ in m.named_parameters()}
    worst = {k: rel(chain.grads[k].reshape(pt[k].shape), pt[k].grad) for k in expected}
    assert max(worst.values()) <= 1e-10, sorted(worst.items(), key=lambda kv: -kv[1])[:4]


def _emulated(monkeypatch, C, heads, shape, bug=None):
    E.install(monkeypatch)
    m, x, G = RP.build(C, heads, shape, cout=2)
    if bug is not None:
        RP.BUGS[bug][0](monkeypatch)
    rec = RP.Recorder(monkeypatch)
    logits, sv, blocks = RP.step(m, x, G, rec, RP.forward_flat)
    return RP.replay(m, x, G, logits, sv, blocks, rec)


EMULATED = {"C12-3heads": (12, 3, (3, 1, 7, 9)), "C100-4heads": (100, 4, (2, 3, 12, 20))}


@pytest.mark.parametrize("geo", sorted(EMULATED))
def test_emulated_stack_passes_every_stage(geo, monkeypatch):
    C, heads, shape = EMULATED[geo]
    mode = _emulated(monkeypatch, C, heads, shape)
    worst = mode.worst_by_kind()
    print("\n".join(f"{k:32s} {v:.3e}" for k, v in sorted(worst.items())))
    assert not mode.failures, "\n".join(mode.failures.values())
    # every stage of both blocks, every parameter and every pad was looked at
    names = set(mode.ratios) | {n for n in mode.failures}
    assert sum(n.startswith("grad ") for n in names) == 7 + 14 * 2
    assert {f"b{b}.{s}" for b in range(2) for s in ("qkv", "o", "du", "dq", "dx_in", "dh_b")} <= names


@pytest.mark.parametrize("bug", sorted(RP.BUGS))
def test_bug_model_fails_its_stage(bug, monkeypatch):
    C, heads, shape = EMULATED["C100-4heads"]
    mode = _emulated(monkeypatch, C, heads, shape, bug)
    failed = mode.failed_kinds()
    print(f"{bug}: {failed}")
    assert RP.BUGS[bug][1] in failed, (bug, failed)
