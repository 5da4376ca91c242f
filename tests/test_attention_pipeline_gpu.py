"""The load pipeline of the tensor-core attention kernels (csrc/pg_attention_tc.cuh): a producer warp runs ahead of
the two consumer warpgroups through a ring of shared-memory stages whose depth differs per <DK, DV> instance, and the
consumers take turns on the tensor cores.  These tests walk the ring: sequence lengths that give 1, 2, depth,
depth + 1 and 2 depth + 1 tiles per CTA (a stage filled once, every stage filled once, the first stage reused, every
stage reused twice and one more), none a multiple of 128, strict and not, and enough (image, head) pairs for several
waves of CTAs.  Every result is held element by element to the float64 bounds of tests/_attention_reference.py, and a
second run on the same inputs must give the same bits."""

import zlib

import pytest
import torch

import _attention_reference as R
from _attention_reference import check, check_equal

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
# ring depth of each <DK, DV> instance (the table above launch_fwd): forward and dQ stage 128-key tiles of K / V,
# dK / dV stages 64-query tiles of Q / dO
DEPTH = {
    (64, 64): dict(fwd=4, dq=4, dkv=4),
    (64, 128): dict(fwd=4, dq=3, dkv=4),
    (128, 64): dict(fwd=4, dq=3, dkv=4),
    (128, 128): dict(fwd=3, dq=2, dkv=4),
}


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _dev():
    return torch.device("cuda:0")


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _counts(depth):
    return {1, 2, depth, depth + 1, 2 * depth + 1}


def ring_lengths(ks, vs):
    """Sequence lengths whose longest CTA walks 1, 2, depth, depth + 1 and 2 depth + 1 tiles of each kernel's ring."""
    d = DEPTH[(ks, vs)]
    key_tiles = _counts(d["fwd"]) | _counts(d["dq"])  # tiles of 128 keys
    query_tiles = _counts(d["dkv"])                   # tiles of 64 queries
    return sorted({128 * c - 37 for c in key_tiles} | {64 * c - 21 for c in query_tiles})


def _slots(x):
    """[N, H, S, d] -> [N * S, H * d] pixel-major."""
    N, H, S, d = x.shape
    return x.permute(0, 2, 1, 3).reshape(N * S, H * d)


def _heads(y, N, H, S, d):
    return y.reshape(N, S, H, d).permute(0, 2, 1, 3)


def _run(L, q, k, v, do, strict, ks, vs):
    """Forward, then backward on the forward's own o and lse, on q | k | v fused as ImageGPT has them; twice, and the
    second run must reproduce the first bit for bit.  Returns o, dq, dk, dv as [N, H, S, d] and lse as [N, H, S]."""
    N, H, S, _ = q.shape
    qkv = torch.cat([_slots(q), _slots(k), _slots(v)], dim=1).contiguous()
    qv, kv, vv = qkv[:, :H * ks], qkv[:, H * ks:2 * H * ks], qkv[:, 2 * H * ks:]
    dov = _slots(do).contiguous()
    runs = []
    for _ in range(2):
        o = torch.full((N * S, H * vs), float("nan"), dtype=BF16, device=_dev())
        dqkv = torch.full_like(qkv, float("nan"))
        lse = torch.full((N, H, S), float("nan"), dtype=F32, device=_dev())
        delta = torch.full((N, H, S), float("nan"), dtype=F32, device=_dev())
        L.causal_attn_fwd(qv, kv, vv, o, lse, N, S, H, ks, vs, strict, impl=0, dk_true=ks)
        L.causal_attn_bwd(qv, kv, vv, o, dov, lse, delta, None, dqkv[:, :H * ks], dqkv[:, H * ks:2 * H * ks],
                          dqkv[:, 2 * H * ks:], N, S, H, ks, vs, strict, impl=0, dk_true=ks)
        torch.cuda.synchronize()
        runs.append((o, lse, delta, dqkv))
    for name, a, b in zip(("o", "lse", "delta", "dq | dk | dv"), *runs):
        check_equal(f"second run, {name}", b, a)
    o, lse, _, dqkv = runs[0]
    return dict(o=_heads(o, N, H, S, vs), lse=lse, dq=_heads(dqkv[:, :H * ks], N, H, S, ks),
                dk=_heads(dqkv[:, H * ks:2 * H * ks], N, H, S, ks), dv=_heads(dqkv[:, 2 * H * ks:], N, H, S, vs))


def _case(L, name, regime, N, H, S, ks, vs, strict):
    q, k, v, do = R.make_inputs(regime, N, H, S, ks, vs, _seed(name), device=_dev())
    ref = R.attention(q, k, v, do, strict, ks, ks, vs)
    got = _run(L, q, k, v, do, strict, ks, vs)
    for t in ("o", "lse", "dq", "dk", "dv"):
        check(f"{name} {t}", got[t], ref[t], ref[f"b_{t}"])


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("ks,vs", list(DEPTH))
def test_ring_walk(L, ks, vs, strict):
    """Every instance at every length of ring_lengths, N = 2, H = 3, scores whose row maximum moves into every key tile
    (`rising`), so a tile read from the wrong stage moves the result far outside its bound."""
    for S in ring_lengths(ks, vs):
        _case(L, f"<{ks},{vs}> S={S} strict={strict}", "rising", 2, 3, S, ks, vs, strict)


def test_ring_lengths_cover_every_depth():
    """The lengths reach each tile count for each kernel of each instance, and none is a multiple of 128."""
    for (ks, vs), d in DEPTH.items():
        lengths = ring_lengths(ks, vs)
        assert all(S % 128 for S in lengths), lengths
        for kernel, tile in (("fwd", 128), ("dq", 128), ("dkv", 64)):
            want = _counts(d[kernel])
            assert want <= {-(-S // tile) for S in lengths}, (ks, vs, kernel, lengths)


@pytest.mark.parametrize("ks,vs", [(64, 64), (128, 128)])
def test_several_waves(L, ks, vs):
    """N = 12, H = 8, S = 603 (five key tiles, ten query tiles): 480 CTAs per kernel, more than three waves on 132 SMs,
    with CTAs of every ring occupancy from one tile to the full walk resident side by side."""
    _case(L, f"<{ks},{vs}> waves", "peaked", 12, 8, 603, ks, vs, False)
