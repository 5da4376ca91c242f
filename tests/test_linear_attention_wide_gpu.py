"""LinearCausalAttention with heads of any width: the chunked scan kernels (pg_linear_attn_fwd / _bwd) against float64
on the GPU, and the module against the oracle.

Kernels.  Each of the four products is written as out_i = x_i . sum_{j <= i} y_j^T z_j (j >= i for dv and dk), and the
reference and the bound both come from cumulative sums of the outer products y_j^T z_j, so memory is O(L d dv), not
O(L^2).  The bound is that of test_conv_path_kernels_gpu.py::test_linear_attention,
  |err| <= (L + max(d, dv) + 2) 2^-24 (tril(|x| |y|^T) |z|)_ic,
element by element.  Outputs are NaN-prefilled, so an element left unwritten fails.

Module.  The oracle runs in float64 on the GPU from the same weights; output, dx and every parameter gradient are
compared relative to max(1, max|ref|): 1e-3 where the 1x1 projections take the fp32 direct kernel, 1e-2 where they take
the bf16 tensor-core GEMM (Cin > 160).
"""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24
F64 = torch.float64
T = 64  # chunk length of the scan kernels


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(dev())


def _within(got, ref, a):
    return bool(((got.to(F64) - ref).abs() <= a).all())


def check(name, got, ref, a):
    """|got - ref| <= a element by element; NaN fails."""
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= a)
    if bad.any():
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound; first at {idx}: "
                             f"got {got[idx].item()!r}, ref {ref[idx].item()!r}, bound {a[idx].item():.3e}")


def _scan64(x, y, z, reverse=False):
    """out_i = x_i . sum_{j <= i} y_j^T z_j (j >= i if reverse) in float64.  x, y: [B, L, P]; z: [B, L, R].  A few
    batch entries at a time, so that the cumulative state holds at most 2^26 elements."""
    if reverse:
        return _scan64(x.flip(1), y.flip(1), z.flip(1)).flip(1)
    step = max(1, (1 << 26) // (x.shape[1] * x.shape[2] * z.shape[2]))
    return torch.cat([torch.einsum("bia,biac->bic", x[b:b + step],
                                   torch.einsum("bja,bjc->bjac", y[b:b + step], z[b:b + step]).cumsum(1))
                      for b in range(0, x.shape[0], step)])


def _products(q, k, v, g):
    """(x, y, z, reverse) of out, dq, dv, dk."""
    return {"out": (q, k, v, False), "dq": (g, v, k, False), "dv": (k, q, g, True), "dk": (v, g, q, True)}


def _segment_positions(B, Lseq, R, sms):
    """Positions per segment of a scan with R output columns: the rule of la_scan in pg_linear_attn.cu (segments only
    when B x 64-column blocks fills at most half of the two-CTAs-per-SM slots, at most one wave, whole chunks)."""
    nch, ctas, slots = math.ceil(Lseq / T), B * math.ceil(R / T), 2 * sms
    nseg = min(nch, slots // ctas) if 2 * ctas <= slots else 1
    return math.ceil(nch / nseg) * T


def _run(L, q, k, v, g):
    out = torch.full(v.shape, float("nan"), device=dev())
    L.linear_attn_fwd(q, k, v, out)
    grads = []
    for _ in range(2):
        dq, dk, dv = (torch.full(t.shape, float("nan"), device=dev()) for t in (q, k, v))
        L.linear_attn_bwd(q, k, v, g, dq, dk, dv)
        grads.append({"dq": dq, "dk": dk, "dv": dv})
    torch.cuda.synchronize()
    return out, grads


def _run_and_check(L, B, Lseq, d, dv, seed):
    """Runs the forward and (twice) the backward on bf16-rounded inputs and checks all four products against the
    float64 reference within the bound, and the two backward runs for identical bits.  Returns the float64 inputs and
    the references."""
    q, k, v, g = (_randn((B, Lseq, n), seed + i).bfloat16().float() for i, n in enumerate((d, d, dv, dv)))
    out, grads = _run(L, q, k, v, g)
    got = {"out": out, **grads[0]}
    t64 = [t.to(F64) for t in (q, k, v, g)]
    prods, prods_abs = _products(*t64), _products(*(t.abs() for t in t64))
    c = (Lseq + max(d, dv) + 2) * U24
    tag = f"linear attention B={B} L={Lseq} d={d} dv={dv}"
    refs = {}
    for name, (x, y, z, rev) in prods.items():
        refs[name] = _scan64(x, y, z, rev)
        xa, ya, za, _ = prods_abs[name]
        check(f"{tag}: {name}", got[name], refs[name], c * _scan64(xa, ya, za, rev))
    for name in ("dq", "dk", "dv"):
        assert torch.equal(grads[0][name].view(torch.int32), grads[1][name].view(torch.int32)), f"{tag}: {name} repeated"
    return t64, refs


@pytest.mark.parametrize("B,Lseq,d,dv", [(1, 1, 128, 128), (2, 63, 65, 64), (2, 65, 128, 128), (3, 784, 256, 64),
                                         (2, 784, 64, 256), (1, 1000, 200, 72), (2, 129, 512, 512)])
def test_linear_attention_wide(L, B, Lseq, d, dv):
    """Heads wider than 64 / 128 channels, widths that are not multiples of the 64-wide tiles, sequences that end
    inside a chunk.  On the shorter sequences the cumulative-sum reference is also checked against autograd of the
    masked O(L^2) form, so the four products are the gradients.  The backward runs twice: identical bits."""
    t64, refs = _run_and_check(L, B, Lseq, d, dv, 4100 + Lseq + 7 * d + dv)
    tag = f"linear attention B={B} L={Lseq} d={d} dv={dv}"
    if Lseq <= 1000:
        q64, k64, v64 = (t.clone().requires_grad_(True) for t in t64[:3])
        mask = torch.tril(torch.ones(Lseq, Lseq, dtype=F64, device=dev()))
        ref = torch.einsum("bij,bjc->bic", torch.einsum("bia,bja->bij", q64, k64) * mask, v64)
        ref.backward(t64[3])
        for name, r in (("out", ref.detach()), ("dq", q64.grad), ("dk", k64.grad), ("dv", v64.grad)):
            assert torch.allclose(refs[name], r, rtol=1e-9, atol=1e-9 * r.abs().max().item()), f"{tag}: {name} reference"


@pytest.mark.parametrize("regime", ["one_segment", "segments_of_several_chunks"])
def test_linear_attention_scan_regimes(L, regime):
    """The two launch shapes in which a CTA carries the state from one chunk to the next (written to the scratch
    buffer after a chunk, read back before the next), with d = 96, dv = 160 (two and three 64-wide passes over the
    state, two and three column blocks).  The batch and length come from the card's SM count, and the regime of each
    scan (R = d for dq and dk, R = dv for out and dv) is asserted:
      one_segment: B x column blocks above the SM count, so every CTA walks the whole sequence (five chunks);
      segments_of_several_chunks: B x column blocks at most the SM count, so the sequence is split into segments of
      at least two chunks, the last segment and the last chunk shorter than the others."""
    d, dv, sms = 96, 160, L.sm_count()
    if regime == "one_segment":
        B, Lseq = sms // 2 + 1, 5 * T - 20
    else:
        B = max(1, sms // 3)
        Lseq = 3 * T * (2 * sms // (B * math.ceil(min(d, dv) / T))) + 17
    for R in (d, dv):
        seg = _segment_positions(B, Lseq, R, sms)
        if regime == "one_segment":
            assert seg >= Lseq > T, (R, seg)
        else:
            assert 2 * T <= seg < Lseq, (R, seg)
    _run_and_check(L, B, Lseq, d, dv, 4700 + len(regime))


def test_linear_attention_long_sequence_segments(L):
    """One image, 16384 positions: the sequence is split into segments that each start from the fixed-order sum of the
    segments before them (after them, for dv and dk).  Self-check: the bound rejects a forward scan whose carry skips
    the segment just before."""
    B, Lseq, d, dv = 1, 16384, 64, 64
    seg = _segment_positions(B, Lseq, dv, L.sm_count())
    assert seg < Lseq, "expected this sequence to be split into segments"
    q, k, v, g = (_randn((B, Lseq, n), 5200 + i).bfloat16().float() for i, n in enumerate((d, d, dv, dv)))
    out, grads = _run(L, q, k, v, g)
    got = {"out": out, **grads[0]}
    t64 = [t.to(F64) for t in (q, k, v, g)]
    prods, prods_abs = _products(*t64), _products(*(t.abs() for t in t64))
    c = (Lseq + max(d, dv) + 2) * U24
    for name, (x, y, z, rev) in prods.items():
        xa, ya, za, _ = prods_abs[name]
        ref, bound = _scan64(x, y, z, rev), c * _scan64(xa, ya, za, rev)
        check(f"L={Lseq}: {name}", got[name], ref, bound)
        if name == "out":
            nseg = math.ceil(Lseq / seg)
            pad = nseg * seg - Lseq
            outer = torch.nn.functional.pad(torch.einsum("bja,bjc->bjac", y, z), (0, 0, 0, 0, 0, pad))
            seg_sums = outer.view(B, nseg, seg, d, dv).sum(2)  # [B, nseg, d, dv]
            prev = torch.cat([torch.zeros_like(seg_sums[:, :1]), seg_sums[:, :-1]], 1)
            prev = prev.repeat_interleave(seg, 1)[:, :Lseq]  # the previous segment's sum at every position
            skipped = ref - torch.einsum("bia,biac->bic", x, prev)
            assert not _within(skipped, ref, bound), "the bound does not detect a carry that skips a segment"
    for name in ("dq", "dk", "dv"):
        assert torch.equal(grads[0][name].view(torch.int32), grads[1][name].view(torch.int32)), f"{name} repeated"


# --------------------------------------------------------------------------------------------------
# LinearCausalAttention against the oracle
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kwargs,shape,tol", [
    (dict(in_channels=128), (2, 128, 28, 28), 1e-3),
    (dict(in_channels=32, n_heads=2, embed_channels=512, out_channels=192), (2, 32, 32, 32), 1e-3),
    (dict(in_channels=256, n_heads=2), (2, 256, 16, 16), 1e-2),
    (dict(in_channels=128), (1, 128, 64, 64), 1e-3),
], ids=["c128_28x28", "c32_h2_e512_o192_32x32", "c256_h2_16x16", "c128_64x64"])
def test_linear_causal_attention_wide_matches_oracle(kwargs, shape, tol):
    """Constructions the 64 / 128-channel kernels refused: one 128-channel head (the module's defaults), d = 256 and
    dv = 96 per head, two 128-channel heads behind bf16 projections, and a 64 x 64 image (L = 4096)."""
    import pytorch_generative_b200 as pg
    from pytorch_generative_b200 import nn  # noqa: F401
    from oracle import reference_path as O

    torch.manual_seed(11)
    m = pg.nn.LinearCausalAttention(**kwargs)
    n_heads = kwargs.get("n_heads", 1)
    embed = kwargs.get("embed_channels") or kwargs["in_channels"]
    out_ch = kwargs.get("out_channels") or kwargs["in_channels"]
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(shape, generator=gen) * 0.5
    dy = torch.randn(shape[0], out_ch, *shape[2:], generator=gen)
    pt = O.trainable({k_: t.detach().to(dev(), F64) for k_, t in m.state_dict().items()})
    xr = x.to(dev(), F64).requires_grad_(True)
    yr = O.linear_causal_attention(xr, pt, "", n_heads, embed, out_ch)
    yr.backward(dy.to(dev(), F64))
    m = m.to(dev())
    xd = x.to(dev()).requires_grad_(True)
    y = m(xd)
    y.backward(dy.to(dev()))

    def close(name, got, ref):
        bound = tol * max(1.0, ref.abs().max().item())
        err = (got.detach().to(F64) - ref.detach()).abs().max().item()
        assert err <= bound and not torch.isnan(got).any(), f"{name}: max err {err:.3e} > {bound:.3e}"

    close("y", y, yr)
    close("dx", xd.grad, xr.grad)
    for name, p in m.named_parameters():
        close("d" + name, p.grad, pt[name].grad)
