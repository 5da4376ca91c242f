"""The pixel-major stacks of GatedPixelCNN, PixelSNAIL, VAE, VQ-VAE and VQ-VAE-2 on the H100, stage by stage
(tests/_conv_stack_reference.py): every convolution's operand, outputs, dx, dw, db and dres, GatedPixelCNN's gates,
direct image convolutions and casts, PixelSNAIL's gated residuals and attention sub-steps, the latent, the quantizer
and the MSE, each against a float64 reference computed from that stage's own recorded inputs with the stage's
per-element bound; every pad column exactly +0.0; every GatedPixelCNN and PixelSNAIL hand-off (each stage's input
against the stage graph, each gradient against what its consumers returned: bit for bit from one, their sum from
several).  Then a second identical step gives identical bits, and the bug models of tests/_conv_stack_replay.py, which
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
    # the recipe model: every 1xN / Nx1 takes the gather path (28 x 28 does not suit the tap loop)
    "gated-recipe-2x1x28x28": ("GatedPixelCNN", dict(in_channels=1, out_channels=1, n_gated=10, gated_channels=128,
                                                     head_channels=32), (2, 1, 28, 28),
                               dict(conv=76, small=3, gate=22, act_cast=1)),
    "gated-tap-loop-2x3x32x32": ("GatedPixelCNN", dict(in_channels=3, out_channels=3, n_gated=2, gated_channels=64,
                                                       head_channels=32), (2, 3, 32, 32),
                                 dict(conv=20, small=3, gate=6, act_cast=1)),
    # the input layer's 1x7 (K = 168) through `pm.conv`; 12 head channels: the logits' operand is padded
    "gated-conv-input-2x24x16x16": ("GatedPixelCNN", dict(in_channels=24, out_channels=24, n_gated=2, gated_channels=64,
                                                          head_channels=12), (2, 24, 16, 16),
                                    dict(conv=21, small=2, gate=6, act_cast=1)),
    "gated-odd-widths-2x1x16x16": ("GatedPixelCNN", dict(in_channels=1, out_channels=2, n_gated=3, gated_channels=20,
                                                         head_channels=12), (2, 1, 16, 16),
                                   dict(conv=27, small=3, gate=8, act_cast=1)),
    # the recipe model: every 2x2 takes the gather path; 4 key channels in a 64-wide slot, 32 value channels in another
    "snail-recipe-2x1x28x28": ("PixelSNAIL", dict(in_channels=1, out_channels=1, n_channels=64, n_pixel_snail_blocks=8,
                                                  n_residual_blocks=2, attention_key_channels=4,
                                                  attention_value_channels=32), (2, 1, 28, 28),
                               dict(conv=58, small=1, gated_res=16, act_cast=8, attention=8)),
    # C4-shaped: 256 channels on the tap loop, 16 key channels, 128 value channels fill their slot
    "snail-c4-2x3x32x32": ("PixelSNAIL", dict(in_channels=3, out_channels=3, n_channels=256, n_pixel_snail_blocks=2,
                                              n_residual_blocks=2, attention_key_channels=16,
                                              attention_value_channels=128), (2, 3, 32, 32),
                           dict(conv=16, small=1, gated_res=4, act_cast=2, attention=2)),
    # 20 channels, 3 key and 12 value channels, 2 outputs: every operand padded, q reads an image column, dy_b padded
    "snail-odd-widths-2x1x16x16": ("PixelSNAIL", dict(in_channels=1, out_channels=2, n_channels=20,
                                                      n_pixel_snail_blocks=1, n_residual_blocks=1,
                                                      attention_key_channels=3, attention_value_channels=12),
                                   (2, 1, 16, 16), dict(conv=7, small=1, gated_res=1, act_cast=1, attention=1)),
    # the input convolution's K = 24 x 9 = 216 through `pm.conv`
    "snail-conv-input-2x24x16x16": ("PixelSNAIL", dict(in_channels=24, out_channels=2, n_channels=20,
                                                       n_pixel_snail_blocks=1, n_residual_blocks=1,
                                                       attention_key_channels=3, attention_value_channels=12),
                                    (2, 24, 16, 16), dict(conv=8, gated_res=1, act_cast=1, attention=1)),
}
# the geometry each bug model runs at: one that runs the code it changes
BUG_GEOMETRY = {None: "vae-recipe-2x1x32x32", "stride4": "vq-vae-recipe-2x3x32x32", "vq": "vq-vae-recipe-2x3x32x32",
                "gated": "gated-recipe-2x1x28x28", "snail": "snail-recipe-2x1x28x28"}


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
    elif key.startswith(("gated-tap-loop", "snail-c4")):
        assert pm.TAP_LOOP in modes, modes
    else:
        assert pm.GATHER in modes, modes


def test_second_step_gives_identical_bits(monkeypatch):
    """Two steps from the same parameters and buffers give the same outputs and gradients, bit for bit (the EMA buffers
    are restored between them)."""
    _two_identical_steps("vq-vae-2-recipe-2x3x32x32")


def test_second_step_gives_identical_bits_gated_pixel_cnn():
    _two_identical_steps("gated-recipe-2x1x28x28")


def test_second_step_gives_identical_bits_pixel_snail():
    _two_identical_steps("snail-recipe-2x1x28x28")


def _two_identical_steps(key):
    cls, kw, shape, _ = GEOMETRIES[key]
    m, x, G = RP.build(cls, kw, shape, device="cuda")
    state = {k: v.clone() for k, v in m.state_dict().items()}
    results = []
    for _ in range(2):
        with torch.no_grad():  # in place: the shape buffers a first forward registers are not in `state`
            for k, t in m.state_dict().items():
                if k in state:
                    t.copy_(state[k])
        out = RP.step(m, x, G)
        # (the last gated layer's vertical 1x1 feeds nothing and gets no gradient)
        results.append(([o.detach().clone() for o in out],
                        {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None},
                        {k: v.clone() for k, v in m.state_dict().items()}))
    (o1, g1, s1), (o2, g2, s2) = results
    assert all(torch.equal(a, b) for a, b in zip(o1, o2))
    assert g1.keys() == g2.keys() and all(torch.equal(g1[n], g2[n]) for n in g1)
    assert all(torch.equal(s1[k], s2[k]) for k in s1)


@pytest.mark.parametrize("bug", sorted(RP.BUGS))
def test_bug_model_fails_its_stage(bug, monkeypatch):
    _, _, _, _, C, _, _ = _run(monkeypatch, BUG_GEOMETRY[RP.BUGS[bug][2]], bug)
    failed = C.failed_kinds()
    print(f"{bug}: {sorted(failed)}")
    assert RP.BUGS[bug][1] in failed, (bug, sorted(failed))
