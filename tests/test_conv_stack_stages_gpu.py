"""The pixel-major stacks of VAE, VQ-VAE and VQ-VAE-2 on the H100, stage by stage (tests/_conv_stack_reference.py):
every convolution's operand, outputs, dx, dw, db and dres, the latent, the quantizer and the MSE, each against a float64
reference computed from that stage's own recorded inputs with the stage's per-element bound; every pad column exactly
+0.0.  Then a second identical step gives identical bits, and the bug models of tests/_conv_stack_replay.py, which
change only which valid tensor or argument the product passes, fail at real sizes on a geometry that runs the code they
change.

Biases are N(0, 0.5^2) and every model output (logits or x_hat, kl or vq_loss) gets a unit-scale cotangent."""

import pytest
import torch

import _conv_stack_replay as RP

pytestmark = pytest.mark.gpu

_VAE = dict(in_channels=1, out_channels=1, latent_channels=16, strides=[2, 2, 2, 2], hidden_channels=64,
            residual_channels=32)
_VQ = dict(in_channels=3, out_channels=3, hidden_channels=128, residual_channels=32, n_residual_blocks=2,
           n_embeddings=512, embedding_dim=64)
_VQ2 = dict(in_channels=3, out_channels=3, hidden_channels=128, n_residual_blocks=2, residual_channels=64,
            n_embeddings=512, embedding_dim=64)
# name -> (model class, constructor keywords, input shape, {stage kind: records})
GEOMETRIES = {
    "vae-recipe-2x1x32x32": ("VAE", _VAE, (2, 1, 32, 32), dict(conv=40, strided=4, transposed=4, latent=1)),
    "vae-odd-widths-2x1x16x16": ("VAE", dict(in_channels=1, out_channels=1, latent_channels=5, strides=[2, 2],
                                             hidden_channels=12, residual_channels=6), (2, 1, 16, 16),
                                 dict(conv=20, strided=2, transposed=2, latent=1)),
    # stride 4: the first transposed convolution emits ReLU
    "vq-vae-recipe-2x3x32x32": ("VectorQuantizedVAE", _VQ, (2, 3, 32, 32),
                                dict(conv=11, strided=2, transposed=2, quantizer=1)),
    # residual width 64 at 16 x 16: the residual 3x3 convolutions of the bottom level take the tap loop
    "vq-vae-2-recipe-2x3x32x32": ("VectorQuantizedVAE2", _VQ2, (2, 3, 32, 32),
                                  dict(conv=23, strided=2, transposed=2, quantizer=2, mse=1)),
}
# the geometry each bug model runs at: one that runs the code it changes
BUG_GEOMETRY = {None: "vae-recipe-2x1x32x32", "stride4": "vq-vae-recipe-2x3x32x32", "vq": "vq-vae-recipe-2x3x32x32"}


def _run(monkeypatch, key, bug=None):
    cls, kw, shape, _ = GEOMETRIES[key]
    m, x, G = RP.build(cls, kw, shape, device="cuda")
    if bug is not None:
        RP.BUGS[bug][0](monkeypatch)
    rec = RP.Recorder(monkeypatch)
    out = RP.step(m, x, G)
    torch.cuda.synchronize()
    C, counts, modes = RP.replay(m, rec)
    return m, x, G, out, C, counts, modes


@pytest.mark.parametrize("key", list(GEOMETRIES))
def test_every_stage_within_its_bound(key, monkeypatch):
    from pytorch_generative_b200.nn import pm

    m, x, G, out, C, counts, modes = _run(monkeypatch, key)
    worst = C.worst_by_kind()
    print(f"\n[{key}] worst |err| / bound per stage")
    print("\n".join(f"  {k:24s} {v:.3e}" for k, v in sorted(worst.items())))
    assert not C.failures, "\n".join(C.failures.values())
    assert counts == GEOMETRIES[key][3], counts
    if key.startswith("vq-vae-2"):
        assert pm.TAP_LOOP in modes and pm.GATHER in modes, modes
    else:
        assert pm.GATHER in modes, modes


def test_second_step_gives_identical_bits(monkeypatch):
    """Two steps from the same parameters and buffers give the same outputs and gradients, bit for bit (the EMA buffers
    are restored between them)."""
    cls, kw, shape, _ = GEOMETRIES["vq-vae-2-recipe-2x3x32x32"]
    m, x, G = RP.build(cls, kw, shape, device="cuda")
    state = {k: v.clone() for k, v in m.state_dict().items()}
    results = []
    for _ in range(2):
        with torch.no_grad():  # in place: the shape buffers a first forward registers are not in `state`
            for k, t in m.state_dict().items():
                if k in state:
                    t.copy_(state[k])
        out = RP.step(m, x, G)
        results.append(([o.detach().clone() for o in out], {n: p.grad.clone() for n, p in m.named_parameters()},
                        {k: v.clone() for k, v in m.state_dict().items()}))
    (o1, g1, s1), (o2, g2, s2) = results
    assert all(torch.equal(a, b) for a, b in zip(o1, o2))
    assert all(torch.equal(g1[n], g2[n]) for n in g1)
    assert all(torch.equal(s1[k], s2[k]) for k in s1)


@pytest.mark.parametrize("bug", sorted(RP.BUGS))
def test_bug_model_fails_its_stage(bug, monkeypatch):
    _, _, _, _, C, _, _ = _run(monkeypatch, BUG_GEOMETRY[RP.BUGS[bug][2]], bug)
    failed = C.failed_kinds()
    print(f"{bug}: {sorted(failed)}")
    assert RP.BUGS[bug][1] in failed, (bug, sorted(failed))
