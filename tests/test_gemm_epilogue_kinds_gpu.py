"""Epilogue kinds of pg_gemm_bf16's tensor-core kernel.  At BN = 128 with K-major A the kernel runs an epilogue built for
the launch's combination of operands (bf16 output with or without bias, bias + GELU and GELU', x a given act', bias
plus one or two fp32 residuals into fp32); every other launch, and every narrower tile, runs the generic epilogue.
Each case is checked at M ending 1, 15, 17, 64 and 127 rows into its last tile, at N ending inside a 32-column group,
with 1, 3 and 5 work items per CTA, for forward (B K-major) and dgrad (B MN-major) operands, into strided outputs whose
padding columns and the rows past M must keep their canary.

Operands are small integers, so every sum is exact in fp32 and the results must equal the float64 reference of
tests/_gemm_reference.py bit for bit (bf16 outputs: its bf16 rounding).  The activation outputs are compared bit for bit
with the same columns computed by the generic epilogue (64-wide launches), and with the SIMT kernel for the generic
activations, which share the per-element arithmetic."""

import pytest
import torch

import _gemm_reference as G

pytestmark = pytest.mark.gpu

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
CANARY = 12288.0  # exact in fp32 and bf16
PAD_COLS, PAD_ROWS = 8, 16

KINDS = ("plain", "bias", "given", "gelu2", "res", "res2")


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _ints(shape, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).to(F32)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _out(M, N, dtype):
    """A canary-filled [M + PAD_ROWS, N + PAD_COLS] buffer and its [M, N] view."""
    buf = torch.full((M + PAD_ROWS, N + PAD_COLS), CANARY, device="cuda:0", dtype=dtype)
    return buf, buf[:M, :N]


def _check_out(buf, M, N, want):
    got = buf[:M, :N].cpu()
    if buf.dtype == BF16:
        assert torch.equal(got, want.to(F32).to(BF16))
    else:
        assert torch.equal(got.to(F64), want)
    assert bool((buf[:, N:].float() == CANARY).all()), "the kernel wrote into the padding columns N..ld"
    assert bool((buf[M:].float() == CANARY).all()), "the kernel wrote rows at or past M"


def _run_kind(L, kind, M, N, K, b_mn, seed):
    """Runs one launch of `kind` and returns {output name: (buffer, float64 expectation or None)} plus its operands."""
    A = _ints((M, K), -3, 3, seed).to(BF16)
    B = _ints((N, K), -3, 3, seed + 1).to(BF16)
    ref, _ = G.reference(A, B)
    dev = torch.device("cuda:0")
    Ad, Bd = A.to(dev), (B.t().contiguous() if b_mn else B).to(dev)
    bias = _ints((N,), -8, 8, seed + 2)
    ops = dict(A=Ad, B=Bd, bias=bias.to(dev))
    kw, outs = {}, {}
    if kind == "plain":
        buf, view = _out(M, N, BF16)
        kw.update(out_bf16=view)
        outs["bf16"] = (buf, ref)
    elif kind == "bias":
        buf, view = _out(M, N, BF16)
        kw.update(bias=ops["bias"], out_bf16=view)
        outs["bf16"] = (buf, ref + bias.to(F64))
    elif kind == "given":
        aux = _ints((M, N), -3, 3, seed + 3)
        buf, view = _out(M, N, BF16)
        kw.update(aux=aux.to(dev, BF16), dact=L.ACT_GIVEN, out_bf16=view)
        outs["bf16"] = (buf, ref * aux.to(F64))
    elif kind == "gelu2":
        gbuf, gview = _out(M, N, BF16)
        dbuf, dview = _out(M, N, BF16)
        kw.update(bias=ops["bias"], act=L.ACT_GELU | L.ACT_STORE_DERIV, out_bf16=gview, out_pre=dview)
        outs["bf16"] = (gbuf, None)
        outs["pre"] = (dbuf, None)
    else:
        r0 = _ints((M, N), -50, 50, seed + 4)
        want = ref + bias.to(F64) + r0.to(F64)
        kw.update(bias=ops["bias"], res0=r0.to(dev))
        if kind == "res2":
            r1 = _ints((M, N), -50, 50, seed + 5)
            want = want + r1.to(F64)
            kw.update(res1=r1.to(dev))
        buf, view = _out(M, N, F32)
        kw.update(out_f32=view)
        outs["f32"] = (buf, want)
    L.gemm(Ad, Bd, M, N, K, b_mn=b_mn, **kw)
    torch.cuda.synchronize()
    return outs, ops, kw


def _gelu2_by_slabs(L, ops, M, N, K, b_mn):
    """GELU and GELU' of the same columns from 64-wide launches (generic epilogue at BN = 64)."""
    g, d = torch.empty(M, N, dtype=BF16), torch.empty(M, N, dtype=BF16)
    for n0 in range(0, N, 64):
        n1 = min(N, n0 + 64)
        Bs = ops["B"][:, n0:n1] if b_mn else ops["B"][n0:n1]
        go = torch.empty(M, n1 - n0, device="cuda:0", dtype=BF16)
        do = torch.empty(M, n1 - n0, device="cuda:0", dtype=BF16)
        L.gemm(ops["A"], Bs, M, n1 - n0, K, b_mn=b_mn, bias=ops["bias"][n0:n1].contiguous(),
               act=L.ACT_GELU | L.ACT_STORE_DERIV, out_bf16=go, out_pre=do)
        torch.cuda.synchronize()
        g[:, n0:n1], d[:, n0:n1] = go.cpu(), do.cpu()
    return g, d


def _check_kind(L, kind, M, N, K, b_mn, seed):
    outs, ops, _ = _run_kind(L, kind, M, N, K, b_mn, seed)
    if kind == "gelu2":
        g, d = _gelu2_by_slabs(L, ops, M, N, K, b_mn)
        for name, want in (("bf16", g), ("pre", d)):
            buf = outs[name][0]
            assert torch.equal(buf[:M, :N].cpu(), want), f"{name} differs from the generic epilogue"
            assert bool((buf[:, N:].float() == CANARY).all()) and bool((buf[M:].float() == CANARY).all())
        return
    for buf, want in outs.values():
        _check_out(buf, M, N, want)


@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
@pytest.mark.parametrize("tail", [1, 15, 17, 64, 127])
@pytest.mark.parametrize("kind", KINDS)
def test_kind_row_and_column_edges(L, kind, tail, b_mn):
    # N = 296: two full 128-wide tiles, then 40 columns ending 8 into a 32-column group
    M, N, K = 128 * 3 + tail, 296, 192
    _check_kind(L, kind, M, N, K, b_mn, 100 + tail)


@pytest.mark.parametrize("items", [1, 3, 5])
@pytest.mark.parametrize("kind", KINDS)
def test_kind_items_per_cta(L, kind, items):
    # K = 64: both consumer warpgroups are in their epilogues at once, warpgroup 0 takes the last item when odd
    N, K = 128, 64
    M = 128 * items * _sms()
    _check_kind(L, kind, M, N, K, False, 200 + items)


@pytest.mark.parametrize("N", [24, 40], ids=["bn32", "bn64"])
@pytest.mark.parametrize("kind", KINDS)
def test_kind_on_narrow_tiles(L, kind, N):
    # the same epilogue operands on the narrower tiles, which run the generic epilogue
    _check_kind(L, kind, 128 * 2 + 17, N, 128, False, 300 + N)


@pytest.mark.parametrize("split_k", [1, 3])
def test_generic_accumulate_and_split_k(L, split_k):
    M, N, K = 128 * 2 + 15, 296, 64 * 6
    A = _ints((M, K), -3, 3, 401).to(BF16)
    B = _ints((N, K), -3, 3, 402).to(BF16)
    ref, _ = G.reference(A, B)
    c0 = _ints((M, N), -8, 8, 403)
    buf, view = _out(M, N, F32)
    view.copy_(c0.to("cuda:0"))
    L.gemm(A.cuda(), B.cuda(), M, N, K, out_f32=view, accumulate=True, split_k=split_k)
    torch.cuda.synchronize()
    _check_out(buf, M, N, ref + c0.to(F64))


@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_generic_alpha_and_bf16_residuals(L, b_mn):
    # alpha != 1 and bf16 residuals are not in any specialised kind: the generic epilogue at BN = 128
    M, N, K = 128 * 2 + 64, 296, 128
    A = _ints((M, K), -3, 3, 501).to(BF16)
    B = _ints((N, K), -3, 3, 502).to(BF16)
    ref, _ = G.reference(A, B)
    dev = torch.device("cuda:0")
    bias = _ints((N,), -8, 8, 503)
    r0, r1 = _ints((M, N), -20, 20, 504), _ints((M, N), -20, 20, 505)
    fbuf, fview = _out(M, N, F32)
    bbuf, bview = _out(M, N, BF16)
    Bd = (B.t().contiguous() if b_mn else B).to(dev)
    L.gemm(A.to(dev), Bd, M, N, K, b_mn=b_mn, bias=bias.to(dev), res0=r0.to(dev, BF16), res1=r1.to(dev, BF16),
           out_f32=fview, out_bf16=bview, alpha=2.0)
    torch.cuda.synchronize()
    want = 2.0 * ref + bias.to(F64) + r0.to(F64) + r1.to(F64)
    _check_out(fbuf, M, N, want)
    _check_out(bbuf, M, N, want)


@pytest.mark.parametrize("act", ["elu", "tanh", "gelu_pre"])
@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_generic_activations_match_the_row_path(L, act, b_mn):
    # ELU, tanh and GELU with the pre-activation stored run the generic epilogue; the SIMT kernel (impl 1) computes
    # the same per-element arithmetic on exact integer sums
    M, N, K = 128 * 2 + 17, 296, 64
    A = _ints((M, K), -1, 1, 601).to(BF16)
    B = _ints((N, K), -1, 1, 602).to(BF16)
    dev = torch.device("cuda:0")
    bias = _ints((N,), -4, 4, 603).to(dev)
    code = {"elu": L.ACT_ELU, "tanh": L.ACT_TANH, "gelu_pre": L.ACT_GELU}[act]
    got, want = [], []
    for impl, dst in ((0, got), (1, want)):
        bbuf, bview = _out(M, N, BF16)
        pbuf, pview = _out(M, N, BF16)
        Bd = (B.t().contiguous() if b_mn and impl == 0 else B).to(dev)
        L.gemm(A.to(dev), Bd, M, N, K, b_mn=b_mn and impl == 0, bias=bias, act=code, out_bf16=bview, out_pre=pview,
               impl=impl)
        torch.cuda.synchronize()
        dst += [bbuf.cpu(), pbuf.cpu()]
    for g, w in zip(got, want):
        assert torch.equal(g, w)
