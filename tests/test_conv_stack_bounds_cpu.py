"""The pixel-major stacks of GatedPixelCNN, PixelSNAIL, VAE, VQ-VAE and VQ-VAE-2 stage by stage, without a GPU
(tests/_conv_stack_reference.py, tests/_conv_stack_replay.py).

1. The stage references, chained in float64 on their own outputs along the stage table, are the restatements of the
   reference models (oracle/reference_path.py for GatedPixelCNN and PixelSNAIL, tests/_vae_reference.py,
   tests/_vq_vae_reference.py): every output and the gradient of every parameter agree to 1e-10 relative.  This holds
   the table (input activations, owned and consumer activations, which stage feeds each input and residual, paddings and
   crops) to the reference independently of the product.
2. The product's own wiring (the models' pixel-major stages, nn/pm.py's autograd Functions, the quantizer, the latent
   and the MSE) runs on fp32 CPU stand-ins of the kernels (tests/_conv_stack_emulation.py), and every stage, parameter
   gradient, pad and GatedPixelCNN or PixelSNAIL hand-off passes the bounds the GPU test holds the kernels to.  The
   geometries take both the tap-loop and the gather path of `_Conv`, channel counts that are not multiples of 8, a
   stride-4 encoder and decoder, GatedPixelCNN and PixelSNAIL input layers on both sides of `small_conv_ok`, and
   PixelSNAIL's 2x2 convolutions on both paths with its strict attention in narrow and filled head slots.
3. Each bug model (tests/_conv_stack_replay.BUGS), applied alone to the emulated stack, fails the stage it names."""

import pytest
import torch

import _conv_stack_emulation as E
import _conv_stack_reference as R
import _conv_stack_replay as RP
import _vae_reference as V
import _vq_vae_reference as VQ
from oracle import reference_path as O

F64 = torch.float64

# name -> (model class, constructor keywords, input shape)
EMULATED = {
    "vae-odd-widths": ("VAE", dict(in_channels=1, out_channels=1, latent_channels=5, strides=[2, 2], hidden_channels=12,
                                   residual_channels=6), (2, 1, 8, 8)),
    "vae-tap-loop": ("VAE", dict(in_channels=1, out_channels=1, latent_channels=4, strides=[2], hidden_channels=64,
                                 residual_channels=64), (1, 1, 32, 32)),
    "vq-vae-stride4": ("VectorQuantizedVAE", dict(in_channels=3, out_channels=3, hidden_channels=16, residual_channels=8,
                                                  n_residual_blocks=2, n_embeddings=10, embedding_dim=6), (2, 3, 8, 8)),
    "vq-vae-2": ("VectorQuantizedVAE2", dict(in_channels=3, out_channels=3, hidden_channels=16, n_residual_blocks=1,
                                             residual_channels=8, n_embeddings=10, embedding_dim=6), (2, 3, 8, 8)),
    # the input layer's three image convolutions on the direct kernel; every 1xN / Nx1 takes the gather path
    "gated-gather": ("GatedPixelCNN", dict(in_channels=1, out_channels=1, n_gated=2, gated_channels=16,
                                           head_channels=8), (2, 1, 8, 8)),
    "gated-tap-loop": ("GatedPixelCNN", dict(in_channels=3, out_channels=3, n_gated=1, gated_channels=64,
                                             head_channels=16), (1, 3, 16, 16)),
    # the input layer's 1x7 (K = 168) through `pm.conv`; 20 gated, 12 head and 2 output channels: every operand padded
    "gated-odd-widths": ("GatedPixelCNN", dict(in_channels=24, out_channels=2, n_gated=2, gated_channels=20,
                                               head_channels=12), (2, 24, 6, 6)),
    # every 2x2 on the gather path; one head of 4 key channels in a 64-wide slot and 8 value channels in another
    "snail-gather": ("PixelSNAIL", dict(in_channels=1, out_channels=1, n_channels=16, n_pixel_snail_blocks=2,
                                        n_residual_blocks=2, attention_key_channels=4, attention_value_channels=8),
                     (2, 1, 8, 8)),
    # 64 channels on a 16 x 8 image: the 2x2 convolutions take the tap loop; the value slot is filled
    "snail-tap-loop": ("PixelSNAIL", dict(in_channels=3, out_channels=3, n_channels=64, n_pixel_snail_blocks=1,
                                          n_residual_blocks=1, attention_key_channels=16,
                                          attention_value_channels=64), (2, 3, 16, 8)),
    # 20 channels, 3 key and 12 value channels, 2 outputs: every operand padded, q reads an image column
    "snail-odd-widths": ("PixelSNAIL", dict(in_channels=1, out_channels=2, n_channels=20, n_pixel_snail_blocks=1,
                                            n_residual_blocks=1, attention_key_channels=3,
                                            attention_value_channels=12), (2, 1, 6, 6)),
    # the input convolution's K = 24 x 9 = 216 through `pm.conv`
    "snail-conv-input": ("PixelSNAIL", dict(in_channels=24, out_channels=2, n_channels=20, n_pixel_snail_blocks=1,
                                            n_residual_blocks=1, attention_key_channels=3,
                                            attention_value_channels=12), (2, 24, 6, 6)),
}
BUG_GEOMETRY = {None: "vq-vae-stride4", "stride4": "vq-vae-stride4", "vq": "vq-vae-stride4", "gated": "gated-gather",
                "snail": "snail-gather"}


@pytest.mark.parametrize("geo", sorted(EMULATED))
def test_stage_chain_matches_the_restatement(geo):
    cls, kw, shape = EMULATED[geo]
    m, x, G = RP.build(cls, kw, shape)
    names = {k for k, _ in m.named_parameters()}
    P = {k: v.detach().to(F64).clone().requires_grad_(k in names) for k, v in m.state_dict().items()}
    x64, G64 = x.to(F64), [g.to(F64) for g in G]
    eps = None
    if cls == "VAE":
        side = shape[2] // 2 ** len(kw["strides"])
        eps = torch.randn(shape[0], kw["latent_channels"], side, side, generator=torch.Generator().manual_seed(5),
                          dtype=F64)
        # without the optimizing executor: profiled runs would change how its scripted latent functions round the
        # fp32 runs of other tests
        with torch.jit.optimized_execution(False):
            ref = V.forward(P, x64, eps, kw["latent_channels"])
    elif cls in ("GatedPixelCNN", "PixelSNAIL"):
        ref = (O.forward("gated_pixel_cnn" if cls == "GatedPixelCNN" else "pixel_snail", P, x64),)
    else:
        ref = (VQ.vq_vae if cls == "VectorQuantizedVAE" else VQ.vq_vae_2)(P, x64)[:2]
    T = R.table(m.state_dict())
    got = (R.graph_chain(T, P, x64),) if cls in ("GatedPixelCNN", "PixelSNAIL") else R.chain(cls, T, P, x64, eps)
    leaves = [P[k] for k in sorted(names)]

    def grads(out):
        total = sum((o * g).sum() for o, g in zip(out, G64))
        # the last gated layer's vertical output feeds nothing: its 1x1 gets no gradient, in the reference as here
        gs = torch.autograd.grad(total, leaves, allow_unused=True)
        return [torch.zeros_like(p) if g is None else g for p, g in zip(leaves, gs)]

    def rel(a, b):
        return float((a - b).abs().max() / b.abs().max()) if b.abs().max() > 0 else float((a - b).abs().max())

    for a, b in zip(got, ref):
        assert rel(a.detach(), b.detach()) <= 1e-10
    with torch.jit.optimized_execution(False):
        ref_grads = grads(ref)
    worst = {k: rel(a, b) for k, a, b in zip(sorted(names), grads(got), ref_grads)}
    assert max(worst.values()) <= 1e-10, sorted(worst.items(), key=lambda kv: -kv[1])[:4]


def _emulated(monkeypatch, geo, bug=None):
    E.install(monkeypatch)
    cls, kw, shape = EMULATED[geo]
    m, x, G = RP.build(cls, kw, shape)
    if bug is not None:
        RP.BUGS[bug][0](monkeypatch)
    rec = RP.Recorder(monkeypatch)
    RP.step(m, x, G)
    return RP.replay(m, rec)


@pytest.mark.parametrize("geo", sorted(EMULATED))
def test_emulated_stack_passes_every_stage(geo, monkeypatch):
    from pytorch_generative_b200.nn import pm

    C, counts, modes = _emulated(monkeypatch, geo)
    print("\n".join(f"{k:24s} {v:.3e}" for k, v in sorted(C.worst_by_kind().items())))
    assert not C.failures, "\n".join(C.failures.values())
    if geo == "vae-tap-loop":
        assert pm.TAP_LOOP in modes and pm.GATHER in modes, modes
    if geo.startswith("gated"):
        assert (pm.TAP_LOOP if geo == "gated-tap-loop" else pm.GATHER) in modes, modes
    if geo.startswith("gated"):  # the input layer's image convolutions: direct kernel or `pm.conv` by K = Cin kh kw
        assert counts["small"] == (2 if geo == "gated-odd-widths" else 3) and counts["act_cast"] == 1, counts
    if geo.startswith("snail"):
        assert (pm.TAP_LOOP if geo == "snail-tap-loop" else pm.GATHER) in modes, modes
        assert counts.get("small", 0) == (0 if geo == "snail-conv-input" else 1), counts
        blocks = {"snail-gather": 2}.get(geo, 1)
        assert counts["attention"] == counts["act_cast"] == blocks and counts["gated_res"] == blocks * (
            2 if geo == "snail-gather" else 1), counts
    assert counts.get("latent", 0) == (1 if geo.startswith("vae") else 0)
    assert counts.get("quantizer", 0) == {"vq-vae-stride4": 1, "vq-vae-2": 2}.get(geo, 0)


@pytest.mark.parametrize("bug", sorted(RP.BUGS))
def test_bug_model_fails_its_stage(bug, monkeypatch):
    C, _, _ = _emulated(monkeypatch, BUG_GEOMETRY[RP.BUGS[bug][2]], bug)
    failed = C.failed_kinds()
    print(f"{bug}: {sorted(failed)}")
    assert RP.BUGS[bug][1] in failed, (bug, sorted(failed))
