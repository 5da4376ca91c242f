"""Kernel tests of softmax attention: pg_causal_attn_fwd / pg_causal_attn_bwd (the tensor-core kernels, impl 0, in all
four <DK, DV> instances, and the SIMT kernels, impl 1, wherever S <= 1024), both delta kernels, and pg_attn_decode (the
one-block kernel and the split kernel with its merge).

Inputs are bf16 and come from the regimes of tests/_attention_reference.py (randn, peaked, rising, sink, diagonal,
ties, extreme), each scaled to the head's true width, so the online softmax's rescaling, masking and underflow paths
all carry weight.  Results are compared element by element with the float64 reference of that module,
|got - ref| <= SAFETY bound, with the bounds derived in its docstring: no term of a bound depends on the largest
element of an output, so an error on a late row, whose output is small, is held to that row's own bound.  A failure
names the worst element.

Operands sit where the models put them: q | k | v as column views of one fused matrix and dq | dk | dv written into
the views of one fused buffer (ImageGPT), or q alone and k | v fused (PixelSNAIL, CausalAttention); o and dO are views
inside wider buffers.  Every buffer starts as NaN, and every byte outside the views a kernel writes must come back with
the same bits."""

import random
import zlib

import pytest
import torch

import _attention_reference as R
from _attention_reference import check, check_equal

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
NAN = float("nan")
INSTANCES = [(64, 64), (64, 128), (128, 64), (128, 128)]  # (q/k slot, v slot): the four <DK, DV> kernel instances


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _dev():
    return torch.device("cuda:0")


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _slot_width(d):
    return 64 if d <= 64 else 128


def _slots(x, slot):
    """[N, H, S, d] -> [N * S, H * slot] pixel-major, each head zero-padded to its slot."""
    N, H, S, d = x.shape
    out = torch.zeros(N, S, H, slot, dtype=x.dtype, device=x.device)
    out[..., :d] = x.permute(0, 2, 1, 3)
    return out.reshape(N * S, H * slot)


def _heads(y, N, H, S, slot):
    """[N * S, H * slot] (a view) -> [N, H, S, slot]."""
    return y.reshape(N, S, H, slot).permute(0, 2, 1, 3)


def _nan_buffer(rows, width, dtype=BF16):
    return torch.full((rows, width), NAN, dtype=dtype, device=_dev())


def _unchanged_outside(name, buf, before, col_ranges):
    """Every column of `buf` outside the (c0, c1) ranges has the bits it had in `before`."""
    keep = torch.ones(buf.shape[1], dtype=torch.bool, device=buf.device)
    for c0, c1 in col_ranges:
        keep[c0:c1] = False
    check_equal(f"{name} outside its views", buf[:, keep], before[:, keep])


def _zero(name, t):
    """Exactly zero by value (a product with a zero operand may carry either sign)."""
    bad = t != 0
    assert not bad.any(), f"{name}: {int(bad.sum())} nonzero elements; first at {tuple(bad.nonzero()[0].tolist())}"


def delta_kernel(N, H, S, vs, ld_o, ld_do):
    """The delta kernel pg_causal_attn_bwd launches, by its own condition: the vector kernel needs a power-of-two
    number of 8-column lanes per slot, pitches that are multiples of 8 and N H S lanes a multiple of 32."""
    lanes = vs // 8
    pow2 = vs % 8 == 0 and 1 <= lanes <= 32 and lanes & (lanes - 1) == 0
    return "vector" if pow2 and ld_o % 8 == 0 and ld_do % 8 == 0 and (N * H * S * lanes) % 32 == 0 else "generic"


# column layouts of q, k, v (and of dq, dk, dv): buffer widths, then (buffer, first column, end column) of each view;
# each buffer has 8 columns past its views, so its pitch stays a multiple of 8
LAYOUTS = {
    "qkv": lambda H, ks, vs: ([H * (2 * ks + vs) + 8],
                              [(0, 0, H * ks), (0, H * ks, 2 * H * ks), (0, 2 * H * ks, H * (2 * ks + vs))]),
    "q_kv": lambda H, ks, vs: ([H * ks + 8, H * (ks + vs) + 8],
                               [(0, 0, H * ks), (1, 0, H * ks), (1, H * ks, H * (ks + vs))]),
}


def _run(L, q, k, v, do, strict, dk_true, ks, vs, impl, layout):
    """pg_causal_attn_fwd, then pg_causal_attn_bwd on the forward's own o and lse, twice: both runs must give the same
    bits, the inputs must be untouched, and nothing outside the output views may be written.  Returns the outputs as
    [N, H, S, slot] (o, dq, dk, dv) and [N, H, S] (lse, delta) tensors."""
    N, H, S, _ = q.shape
    P = N * S
    widths, spec = LAYOUTS[layout](H, ks, vs)
    ins = [_nan_buffer(P, w) for w in widths]
    grads = [_nan_buffer(P, w) for w in widths]
    qv, kv, vv = (ins[b][:, c0:c1] for b, c0, c1 in spec)
    dqv, dkv, dvv = (grads[b][:, c0:c1] for b, c0, c1 in spec)
    qv.copy_(_slots(q, ks))
    kv.copy_(_slots(k, ks))
    vv.copy_(_slots(v, vs))
    ob, dob = _nan_buffer(P, H * vs + 24), _nan_buffer(P, H * vs + 24)
    ov, dov = ob[:, 8:8 + H * vs], dob[:, 8:8 + H * vs]
    dov.copy_(_slots(do, vs))
    lse = torch.full((N, H, S), NAN, dtype=F32, device=_dev())
    delta = torch.full((N, H, S), NAN, dtype=F32, device=_dev())
    before = [t.clone() for t in (*ins, dob, ob, *grads)]
    runs = []
    for _ in range(2):
        L.causal_attn_fwd(qv, kv, vv, ov, lse, N, S, H, ks, vs, strict, impl=impl, dk_true=dk_true)
        L.causal_attn_bwd(qv, kv, vv, ov, dov, lse, delta, None, dqv, dkv, dvv, N, S, H, ks, vs, strict, impl=impl,
                          dk_true=dk_true)
        torch.cuda.synchronize()
        runs.append([t.clone() for t in (ob, lse, delta, *grads)])
    for i, (a, b) in enumerate(zip(*runs)):
        check_equal(f"impl {impl} second run, output {i}", b, a)
    for i, (t, t0) in enumerate(zip((*ins, dob), before)):
        check_equal(f"impl {impl} input buffer {i}", t, t0)
    _unchanged_outside(f"impl {impl} o buffer", ob, before[len(ins) + 1], [(8, 8 + H * vs)])
    for i, g in enumerate(grads):
        _unchanged_outside(f"impl {impl} gradient buffer {i}", g, before[len(ins) + 2 + i],
                           [(c0, c1) for b, c0, c1 in spec if b == i])
    return dict(o=_heads(ov, N, H, S, vs), lse=lse, delta=delta, dq=_heads(dqv, N, H, S, ks),
                dk=_heads(dkv, N, H, S, ks), dv=_heads(dvv, N, H, S, vs), ld_o=ob.stride(0), ld_do=dob.stride(0))


def _check_run(name, got, ref, do, strict, dk, dv):
    """o, lse and the gradients within their bounds (tests/_attention_reference.py); the padded slot columns of o, dq,
    dk and dv exactly zero; a strict row 0 exactly o = 0, lse = 0, dq = 0.  delta against sum_d dO_id o~_id in float64
    over the kernel's own bf16 o~: an fp32 sum of dv_slot products, so |delta - ref| <= dv_slot U23 sum_d |dO_id o~_id|
    (any summation order; U23 as everywhere)."""
    check(f"{name} o", got["o"][..., :dv], ref["o"], ref["b_o"])
    check(f"{name} lse", got["lse"], ref["lse"], ref["b_lse"])
    for g, d in (("dq", dk), ("dk", dk), ("dv", dv)):
        check(f"{name} {g}", got[g][..., :d], ref[g], ref[f"b_{g}"])
    for t, d in (("o", dv), ("dq", dk), ("dk", dk), ("dv", dv)):
        _zero(f"{name} {t} padded slot columns", got[t][..., d:])
    if strict:
        _zero(f"{name} strict row 0 of o", got["o"][:, :, 0])
        _zero(f"{name} strict row 0 of dq", got["dq"][:, :, 0])
        _zero(f"{name} strict row 0 of lse", got["lse"][:, :, 0])
    vs = got["o"].shape[-1]
    o_k = got["o"].to(F64)
    do64 = torch.zeros_like(o_k)
    do64[..., :dv] = do.to(F64)
    check(f"{name} delta", got["delta"], (do64 * o_k).sum(-1), vs * R.U23 * (do64 * o_k).abs().sum(-1))


def _attention_case(L, name, regime, N, H, S, dk, dv, strict, layout, seed):
    ks, vs = _slot_width(dk), _slot_width(dv)
    q, k, v, do = R.make_inputs(regime, N, H, S, dk, dv, seed, device=_dev())
    ref = R.attention(q, k, v, do, strict, dk, ks, vs)
    for impl in ((0, 1) if S <= 1024 else (0,)):
        got = _run(L, q, k, v, do, strict, dk, ks, vs, impl, layout)
        _check_run(f"{name} impl {impl}", got, ref, do, strict, dk, dv)
    return got


# ----------------------------------------------------------------------------------------------------------------------
# forward and backward
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("regime", R.REGIMES)
@pytest.mark.parametrize("ks,vs", INSTANCES)
def test_instance_regime(L, ks, vs, regime, strict):
    """Every <DK, DV> instance under every input regime, N = 2, H = 2, S = 300 (two full key tiles and a partial one),
    heads 16 and 8 columns narrower than their slots.  Non-strict runs on ImageGPT's fused q | k | v, strict on the
    separate q and fused k | v.  Bounds: tests/_attention_reference.py; delta: _check_run."""
    _attention_case(L, f"<{ks},{vs}> {regime} strict={strict}", regime, 2, 2, 300, ks - 16, vs - 8, strict,
                    "q_kv" if strict else "qkv", _seed(ks, vs, regime, strict))


SWEEP_S = [1, 2, 63, 64, 65, 127, 128, 129, 255, 257, 1000, 1023, 1024, 1025, 4096]
SWEEP_HEADS = [(16, 64), (40, 100), (64, 48), (72, 128), (128, 16)]  # (dk_true, dv_true): slots 64 and 128 each


@pytest.mark.parametrize("regime", ["randn", "peaked", "diagonal"])
@pytest.mark.parametrize("i,S", list(enumerate(SWEEP_S)))
def test_shape_sweep(L, i, S, regime):
    """Sequence lengths around every tile edge of the kernels (64-query tiles of the backward, 128-row tiles elsewhere),
    past the SIMT limit (1024) and at 64x64 images (4096), N = H = 1, the head widths cycling through
    SWEEP_HEADS, strict on every other length.  With N H S odd the backward takes the generic delta kernel.  Bounds:
    tests/_attention_reference.py; delta: _check_run."""
    dk, dv = SWEEP_HEADS[i % len(SWEEP_HEADS)]
    strict = i % 2 == 1
    got = _attention_case(L, f"S={S} dk={dk} dv={dv} {regime} strict={strict}", regime, 1, 1, S, dk, dv, strict,
                          ("qkv", "q_kv")[(i // 2) % 2], _seed(S, regime))
    kind = delta_kernel(1, 1, S, _slot_width(dv), got["ld_o"], got["ld_do"])
    if S % 2:
        assert kind == "generic", f"S={S}: an odd N H S must take the generic delta kernel, not the {kind} one"


def test_sweep_reaches_both_delta_kernels():
    """The sweep's cases reach the vector delta kernel with v slots of 64 and of 128, and the generic kernel."""
    reached = set()
    for i, S in enumerate(SWEEP_S):
        vs = _slot_width(SWEEP_HEADS[i % len(SWEEP_HEADS)][1])
        reached.add((delta_kernel(1, 1, S, vs, vs + 24, vs + 24), vs))
    assert {("vector", 64), ("vector", 128)} <= reached and {("generic", 64), ("generic", 128)} & reached, reached


def test_several_ctas_per_sm(L):
    """N = 12, H = 4, S = 1024: 384 CTAs per kernel, about three waves on 132 SMs, peaked scores.  Bounds:
    tests/_attention_reference.py; delta: _check_run."""
    _attention_case(L, "N=12 H=4 S=1024", "peaked", 12, 4, 1024, 64, 64, False, "qkv", _seed("waves"))


@pytest.mark.parametrize("ks,vs", INSTANCES)
def test_single_position_is_v(L, ks, vs):
    """S = 1, not strict: the only key has p = 1 exactly, so o is v bit for bit, in every instance and both impls."""
    N, H = 3, 2
    q, k, v, do = R.make_inputs("randn", N, H, 1, ks, vs, _seed("one", ks, vs), device=_dev())
    for impl in (0, 1):
        got = _run(L, q, k, v, do, False, ks, ks, vs, impl, "qkv")
        check_equal(f"<{ks},{vs}> impl {impl} o", got["o"].contiguous(), v)


# ----------------------------------------------------------------------------------------------------------------------
# KV-cached decode
# ----------------------------------------------------------------------------------------------------------------------
DECODE_CONFIGS = {
    # strict, H, dk_true, dv_true; q / k / v slots 64
    "pixelsnail": (True, 1, 16, 64),   # q alone, k | v as column views of one fused row matrix
    "imagegpt": (False, 4, 48, 40),    # q | k | v as column views of one fused row matrix
}


@pytest.mark.parametrize("regime", ["peaked", "rising", "sink"])
@pytest.mark.parametrize("S", [300, 1024, 1025, 2048, 3000, 4096])
@pytest.mark.parametrize("config", list(DECODE_CONFIGS))
def test_decode(L, config, S, regime):
    """pg_attn_decode on the one-block path (S <= 1024) and the split path with its merge, at positions on both sides
    of every tile and split edge, the last one and two seeded ones, in PixelSNAIL's and ImageGPT's configurations
    (heads narrower than their 64-wide slots, the scale from dk_true).  Before each step the caches hold the sequence's
    rows below pos and NaN from pos on, in buffers wider than H * slot: a finite result within the forward bound
    (tests/_attention_reference.py, T_i tiles >= the splits, whose merge factors are alphas) shows no row past pos is
    read.  Row pos must then hold k_new / v_new bit for bit and every other byte of the cache buffers be unchanged.  A
    strict step at pos 0 has no keys and gives exactly 0.  `rising` puts the max in the last split, so the merge scales
    the earlier ones by f << 1; `sink` keeps it in split 0."""
    strict, H, dk, dv = DECODE_CONFIGS[config]
    ks = vs = 64
    N = 2
    q, k, v, _ = R.make_inputs(regime, N, H, S, dk, dv, _seed(config, S, regime), device=_dev())
    qs, kss, vss = (_slots(t, w).view(N, S, H * w) for t, w in ((q, ks), (k, ks), (v, vs)))
    if config == "imagegpt":
        rows = [_nan_buffer(N, H * (2 * ks + vs) + 8)]
        qrow, knew, vnew = rows[0][:, :H * ks], rows[0][:, H * ks:2 * H * ks], rows[0][:, 2 * H * ks:H * (2 * ks + vs)]
    else:
        rows = [_nan_buffer(N, H * ks + 8), _nan_buffer(N, H * (ks + vs) + 8)]
        qrow, knew, vnew = rows[0][:, :H * ks], rows[1][:, :H * ks], rows[1][:, H * ks:H * (ks + vs)]
    kcb, vcb = _nan_buffer(N * S, H * ks + 8), _nan_buffer(N * S, H * vs + 16)
    kc, vc = kcb[:, :H * ks], vcb[:, :H * vs]
    ob = _nan_buffer(N, H * vs + 16)
    ov = ob[:, 8:8 + H * vs]
    pos_d = torch.zeros(1, dtype=torch.int32, device=_dev())
    sample = random.Random(_seed(config, S, regime)).sample(range(S), 2)
    positions = sorted({p for p in (0, 1, 127, 128, 1023, 1024, 1025, S - 1, *sample) if p < S})
    filled = 0
    for p in positions:
        kcb.view(N, S, -1)[:, filled:p, :H * ks] = kss[:, filled:p]
        vcb.view(N, S, -1)[:, filled:p, :H * vs] = vss[:, filled:p]
        qrow.copy_(qs[:, p])
        knew.copy_(kss[:, p])
        vnew.copy_(vss[:, p])
        pos_d.fill_(p)
        before = [t.clone() for t in (kcb, vcb, ob, *rows)]
        L.attn_decode(qrow, knew, vnew, kc, vc, ov, pos_d, N, S, H, ks, vs, strict, dk_true=dk)
        torch.cuda.synchronize()
        name = f"{config} S={S} {regime} pos {p}"
        want_k, want_v = before[0].clone(), before[1].clone()
        want_k.view(N, S, -1)[:, p, :H * ks] = kss[:, p]
        want_v.view(N, S, -1)[:, p, :H * vs] = vss[:, p]
        check_equal(f"{name} k cache", kcb, want_k)
        check_equal(f"{name} v cache", vcb, want_v)
        for i, t in enumerate(rows):
            check_equal(f"{name} input rows {i}", t, before[3 + i])
        _unchanged_outside(f"{name} o buffer", ob, before[2], [(8, 8 + H * vs)])
        out = ov.reshape(N, H, vs)
        ref, bound = R.decode_row(q[:, :, p], k, v, p, strict, dk, ks)
        check(name, out[..., :dv], ref, bound)
        _zero(f"{name} padded slot columns", out[..., dv:])
        if strict and p == 0:
            _zero(f"{name} (no keys)", out)
        filled = p + 1
