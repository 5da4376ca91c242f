"""Host-side primitives on pixel-major tensors (thin, allocation + one C-ABI call each).

Everything the model stacks and nn modules do on the device goes through these helpers, which only
allocate outputs and forward to `_lib` (libpg_b200.so).  There is no autograd here: forward and backward
are explicit functions, composed by the `torch.autograd.Function`s in `nn/` and `models/`.

Conventions: `P` = N*H*W pixels; activations are [P, C] row-major ("pixel-major", i.e. NHWC); GEMM
operands are bf16, the residual stream and all gradients that are summed are fp32.
"""

import os

import torch
from torch.utils.weak import WeakIdKeyDictionary, WeakIdRef

from . import _lib as L

BF16 = torch.bfloat16
F32 = torch.float32

# 0 = tensor-core kernels (product); 1 = SIMT cross-check kernels (tests/debug only, set by tests).
ATTN_IMPL = int(os.environ.get("PG_ATTN_IMPL", "0"))
GEMM_IMPL = int(os.environ.get("PG_GEMM_IMPL", "0"))

KERNEL_SLOTS = (64, 128)  # column widths of the attention kernels' head slots, for q/k and for v independently


def head_slots(dk, dv):
    """(q/k slot, v slot) widths for heads with dk query/key and dv value channels: for each, the smallest kernel slot
    that holds the head.  Narrower heads live in zero-padded slots; the scale stays 1/sqrt(dk)."""
    def slot(d, what):
        for s in KERNEL_SLOTS:
            if d <= s:
                return s
        raise NotImplementedError(f"attention: {what}={d} channels per head exceed the widest kernel head slot "
                                  f"({KERNEL_SLOTS[-1]})")
    return slot(dk, "dk"), slot(dv, "dv")


def empty(shape, dtype, like):
    return torch.empty(shape, dtype=dtype, device=like.device)


def zeros(shape, dtype, like):
    return torch.zeros(shape, dtype=dtype, device=like.device)


def round_up(v, m):
    return (v + m - 1) // m * m


def to_bf16(t):
    """fp32 -> bf16 copy through pg_cast_f32_to_bf16 (weights packing)."""
    t = t.contiguous()
    out = torch.empty(t.shape, dtype=BF16, device=t.device)
    L.cast_bf16(t.view(-1), out.view(-1))
    return out


_COPIES = WeakIdKeyDictionary()  # first source -> {key: (weakrefs to the other sources, the signature, the copy)}


def cached_copy(sources, key, build):
    """`build()`, memoised: bf16 copies of fp32 weights are made once per optimizer step, not once per forward.  An
    entry holds while every source is the same object with the same `_version`, `data_ptr()` and shape, and dies with
    `sources[0]`.  A miss builds a new copy (a pending backward keeps reading the old one).  Under CUDA-graph capture
    nothing is returned or stored, so every replay casts.  Whatever writes a source behind autograd's back must call
    `torch.autograd.graph.increment_version` on it (`optim.FusedAdam`, `GraphedTrainStep` after a replay,
    `parallel.broadcast_parameters`), except `CausalConv2d.apply_mask`: it runs before anything copies the weight, and
    only re-zeroes taps that a version-moving write changed since the last copy."""
    if sources[0].is_cuda and torch.cuda.is_current_stream_capturing():
        return build()
    sig = [(s._version, s.data_ptr(), s.shape) for s in sources]
    hit = _COPIES.get(sources[0], {}).get(key)
    if hit is not None and hit[1] == sig and all(r() is s for r, s in zip(hit[0], sources[1:])):
        return hit[2]
    copy = build()
    _COPIES.setdefault(sources[0], {})[key] = (tuple(WeakIdRef(s) for s in sources[1:]), sig, copy)
    return copy


def pack_taps(weight, cin_p, positions=None, cout_p=None):
    """[Cout, Cin, kh, kw] fp32 -> [Cout, T * cin_p] bf16 GEMM operand, tap-major: the columns of kernel position
    t = (i, j) are [t * cin_p, (t + 1) * cin_p), zero beyond Cin.  positions: the (i, j) to pack, in column order;
    None = every kernel position, row-major (pg_tap_gather's K order; a 1x1 conv is the single position (0, 0)).
    cout_p: pad the rows to this many with zeros (an output of exactly zero pad columns); None = Cout rows."""
    def build():
        cout, cin, kh, kw = weight.shape
        w = weight.detach().permute(0, 2, 3, 1).reshape(cout, kh * kw, cin)
        if positions is not None:
            w = w[:, [i * kw + j for i, j in positions]]
        if cin_p != cin:
            w = torch.nn.functional.pad(w, (0, cin_p - cin))
        if cout_p is not None and cout_p != cout:
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, cout_p - cout))
        return to_bf16(w.reshape(w.shape[0], -1))
    key = ("taps", cin_p, None if positions is None else tuple(positions))
    return cached_copy((weight,), key if cout_p is None else key + (cout_p,), build)


def pack_taps_t(weight, cin_p, cout_p):
    """ConvTranspose2d's [Cin, Cout, kh, kw] fp32 -> [T * cout_p, cin_p] bf16 GEMM operand, tap-major rows: the rows of
    kernel position t = (i, j) (row-major, pg_strided_scatter's tap order) are [t * cout_p, (t + 1) * cout_p), zero
    beyond Cout, and its columns are zero beyond Cin.  X [P, cin_p] @ this^T is Y_cat [P, T * cout_p]."""
    def build():
        cin, cout, kh, kw = weight.shape
        w = weight.detach().permute(2, 3, 1, 0)  # [kh, kw, Cout, Cin]
        w = torch.nn.functional.pad(w, (0, cin_p - cin, 0, cout_p - cout))
        return to_bf16(w.reshape(kh * kw * cout_p, cin_p))
    return cached_copy((weight,), ("taps_t", cin_p, cout_p), build)


def padded_bias(bias, n):
    """fp32 bias zero-padded to n entries (the GEMM epilogue reads n); the bias itself when it has n already."""
    b = bias.detach()
    if b.numel() == n:
        return b

    def build():
        out = torch.zeros(n, dtype=F32, device=b.device)
        out[: b.numel()].copy_(b)
        return out
    return cached_copy((bias,), ("pad", n), build)


def nchw_to_pm(x, dtype, width=None):
    """[N, C, H, W] fp32 -> [N*H*W, width>=C] pixel-major (extra columns zero)."""
    x = x.contiguous()
    if x.dtype != F32:
        x = x.float()
    n, c, h, w = x.shape
    width = width or c
    if width == c:
        out = torch.empty(n * h * w, c, dtype=dtype, device=x.device)
        L.nchw_to_pm(x, out)
    else:
        out = torch.zeros(n * h * w, width, dtype=dtype, device=x.device)
        L.nchw_to_pm(x, out[:, :c])
    return out


def pm_to_nchw(x_pm, n, c, h, w, act=L.ACT_NONE):
    out = torch.empty(n, c, h, w, dtype=F32, device=x_pm.device)
    L.pm_to_nchw(x_pm[:, :c] if x_pm.shape[1] != c else x_pm, out, act=act)
    return out


# --------------------------------------------------------------------------------------------------
# Linear (1x1 conv) forward / dgrad / wgrad on pixel-major activations
# --------------------------------------------------------------------------------------------------
SKINNY_ROWS = 32             # the skinny GEMM (pg_gemm_bf16 impl 2) keeps one accumulator per row in each lane
SKINNY_SMEM = 160 * 1024     # ... and stages all of A ([rows, K] bf16) in this much shared memory


def linear_impl(rows, k, skinny):
    """pg_gemm_bf16 implementation of a forward contraction of a [rows, k] operand.  `skinny` asks for the skinny
    kernel (impl 2); it gets it wherever that kernel takes the operands: at most SKINNY_ROWS rows, k % 8 == 0 and A
    within SKINNY_SMEM.  Every other contraction runs on the tensor-core GEMM (GEMM_IMPL: impl 0, any M and K)."""
    if skinny and rows <= SKINNY_ROWS and k % 8 == 0 and rows * k * 2 <= SKINNY_SMEM:
        return 2
    return GEMM_IMPL


def linear_fwd(a, w, bias=None, *, act=L.ACT_NONE, res0=None, res1=None, want_bf16=True, want_pre=False,
               want_f32=False, n_out=None, skinny=False, pre_deriv=False):
    """y = a @ w.T (+bias) (+res0 +res1).  a: [P, K] bf16, w: [Cout, K] bf16.
    Returns (out_bf16 = act(pre), out_pre = bf16(pre), out_f32 = pre), each None unless requested.
    pre_deriv: out_pre holds act'(pre) instead (consumed by linear_dgrad(dact=L.ACT_GIVEN)).
    skinny: run on the skinny kernel where it takes the operands (`linear_impl`)."""
    P, K = a.shape
    n = n_out or w.shape[0]
    ob = empty((P, n), BF16, a) if want_bf16 else None
    op = empty((P, n), BF16, a) if want_pre else None
    of = empty((P, n), F32, a) if want_f32 else None
    L.gemm(a, w, P, n, K, bias=bias, res0=res0, res1=res1, out_bf16=ob, out_pre=op, out_f32=of,
           act=(act | L.ACT_STORE_DERIV) if (pre_deriv and want_pre) else act,
           impl=linear_impl(P, K, skinny))
    return ob, op, of


def linear_dgrad(dy, w, *, aux=None, dact=L.ACT_NONE, want_f32=False, k_in=None):
    """dx = dy @ w (optionally * act'(aux)).  dy: [P, Cout] bf16, w: [Cout, Cin] bf16 (read MN-major)."""
    P, cout = dy.shape
    cin = k_in or w.shape[1]
    ob = empty((P, cin), BF16, dy)
    of = empty((P, cin), F32, dy) if want_f32 else None
    L.gemm(dy, w[:, :cin], P, cin, min(cout, w.shape[0]), b_mn=True, aux=aux, dact=dact, out_bf16=ob, out_f32=of,
           impl=GEMM_IMPL)
    return (ob, of) if want_f32 else ob


def _split_k_for(m_out, n_out, k):
    """Split-K factor of a wgrad GEMM: the largest one whose work items (output tiles x splits) still fit ONE wave of
    the persistent grid.  Rounding up instead (e.g. 32 tiles x 5 = 160 items on 132 SMs) makes a few CTAs run two
    items back to back, so the launch lasts two split-lengths instead of one.  Tiles are 128 x 128 (pg_gemm.cu)."""
    tiles = ((m_out + 127) // 128) * ((n_out + 127) // 128)
    sms = L.sm_count()
    if os.environ.get("PG_SPLITK_ROUND_UP") == "1":  # previous heuristic, kept for A/B runs
        want = max(1, (sms + tiles - 1) // tiles)
    else:
        want = max(1, sms // tiles)
    k_iters = (k + 63) // 64
    return max(1, min(want, k_iters // 8 if k_iters >= 16 else 1))


def linear_wgrad(dy, a, dw_out, db_out=None):
    """dw_out[Cout, Cin] += dy.T @ a over the pixel dimension, split along pixels: each split's fp32 slice goes to scratch
    and the slices are added to dw_out in a fixed order (pg_sum_partials), so the result is the same on every run.
    db_out (fp32 [Cout], pre-zeroed or holding a running sum): += column sums of dy, reduced by the same launch from the
    dy tiles it stages anyway (the bias gradient without a second pass over dy)."""
    P, cout = dy.shape
    cin = a.shape[1]
    assert dw_out.dtype == F32 and dw_out.shape[0] >= cout
    if db_out is not None and GEMM_IMPL != 0:   # the SIMT cross-check build of the stacks: separate column sums
        L.colsum(dy, db_out, accumulate=True)
        db_out = None
    L.gemm(dy, a, cout, cin, P, a_mn=True, b_mn=True, out_f32=dw_out, accumulate=True,
           split_k=_split_k_for(cout, cin, P), impl=GEMM_IMPL, bias_grad=db_out)


# --------------------------------------------------------------------------------------------------
# Tap-loop convolutions (im2col-free): the shifted operand is read in place through 4-D TMA boxes
# --------------------------------------------------------------------------------------------------
def conv_fwd(x, wcat, bias, n_img, h, w, taps, *, act=L.ACT_NONE, res0=None, res1=None, want_bf16=True, want_pre=False,
             want_f32=False, pre_deriv=False):
    """y[p] = bias + sum_t W_t . x[p + taps[t]] (zero outside the image).  x: [P, C] bf16 (C % 64 == 0),
    wcat: [Cout, T*C] bf16 with tap-major columns.  Outputs as linear_fwd."""
    P, C = x.shape
    n = wcat.shape[0]
    ob = empty((P, n), BF16, x) if want_bf16 else None
    op = empty((P, n), BF16, x) if want_pre else None
    of = empty((P, n), F32, x) if want_f32 else None
    L.gemm_conv(x, wcat, P, n, len(taps) * C, L.CONV_FWD, n_img, h, w, C, taps, bias=bias, res0=res0, res1=res1,
                out_bf16=ob, out_pre=op, out_f32=of, act=(act | L.ACT_STORE_DERIV) if (pre_deriv and want_pre) else act)
    return ob, op, of


def conv_dgrad(dy, wcat, cin, n_img, h, w, taps, *, aux=None, dact=L.ACT_NONE, want_f32=False, want_bf16=True, res0=None):
    """dx[p] = sum_t W_t^T . dy[p - taps[t]] (optionally * act'(aux), + res0).  dy: [P, Cout] bf16 (Cout % 64 == 0),
    wcat: [Cout, T*cin] bf16."""
    P, cout = dy.shape
    ob = empty((P, cin), BF16, dy) if want_bf16 else None
    of = empty((P, cin), F32, dy) if want_f32 else None
    L.gemm_conv(dy, wcat, P, cin, len(taps) * cout, L.CONV_DGRAD, n_img, h, w, cout, [(-a, -b) for a, b in taps], aux=aux,
                dact=dact, res0=res0, out_bf16=ob, out_f32=of)
    return ob, of


def conv_wgrad(dy, x, dw_out, n_img, h, w, taps, db_out=None):
    """dw_out[Cout, T*C] += sum_p dy[p]^T . x[p + taps[t]] (fp32 accumulation, split along pixels); db_out as in
    linear_wgrad."""
    P, cout = dy.shape
    C = x.shape[1]
    T = len(taps)
    assert dw_out.dtype == F32 and dw_out.shape[0] >= cout and dw_out.shape[1] == T * C
    bn = 256 if C % 256 == 0 else (128 if C % 128 == 0 else 64)
    tiles = ((cout + 127) // 128) * (T * C // bn)
    k_iters = (P + 63) // 64
    split = max(1, min(max(1, L.sm_count() // tiles), k_iters // 8 if k_iters >= 16 else 1))
    L.gemm_conv(dy, x, cout, T * C, P, L.CONV_WGRAD, n_img, h, w, C, taps, out_f32=dw_out, accumulate=True, split_k=split,
                bias_grad=db_out)


def bias_grad(dy, out=None):
    """Column sums of dy [P, C] into a fp32 [C] vector."""
    C = dy.shape[1]
    if out is None:
        out = torch.zeros(C, dtype=F32, device=dy.device)
    L.colsum(dy, out, accumulate=True)
    return out


# --------------------------------------------------------------------------------------------------
# LayerNorm
# --------------------------------------------------------------------------------------------------
def layernorm_fwd(x, gamma, beta, eps, want_bf16=True, want_f32=False):
    """LayerNorm of the gamma.numel() first columns of x [P, C]; the outputs have x's width, zero beyond gamma's."""
    P, C = x.shape
    yb = empty((P, C), BF16, x) if want_bf16 else None
    yf = empty((P, C), F32, x) if want_f32 else None
    mean = empty((P,), F32, x)
    rstd = empty((P,), F32, x)
    L.layernorm_fwd(x, gamma, beta, eps, y_bf16=yb, y_f32=yf, mean=mean, rstd=rstd)
    return yb, yf, mean, rstd


def layernorm_bwd(dy, x, gamma, mean, rstd, dres0=None, dres1=None, want_bf16=True, want_f32=True, want_colsum=False,
                  stats=None):
    """Returns (dx_f32 (+dres0+dres1), dx_bf16, dgamma, dbeta[, colsum(dx)]).  `stats`: optional zero-filled fp32 [3, C]
    (a slice of the caller's gradient arena) that receives dgamma, dbeta and the column sums.  C = gamma.numel(); x and
    the gradients may be wider (padded columns: dx is zero there)."""
    P, ld = x.shape
    C = gamma.numel()
    dxf = empty((P, ld), F32, x) if want_f32 else None
    dxb = empty((P, ld), BF16, x) if want_bf16 else None
    if stats is None:
        stats = zeros((3, C), F32, x)  # dgamma, dbeta, column sums of dx: one memset
    L.layernorm_bwd(dy, x, gamma, mean, rstd, dres0=dres0, dres1=dres1, dx_f32=dxf, dx_bf16=dxb, dgamma=stats[0],
                    dbeta=stats[1], dx_colsum=stats[2] if want_colsum else None)
    if want_colsum:
        return dxf, dxb, stats[0], stats[1], stats[2]
    return dxf, dxb, stats[0], stats[1]


# --------------------------------------------------------------------------------------------------
# Attention on padded head slots (widths from head_slots)
# --------------------------------------------------------------------------------------------------
def attn_fwd(q, k, v, n_img, seq, heads, dk_true, qk_slot, dv_slot, strict):
    """q, k: [P, heads*qk_slot] bf16 (dk_true valid columns per slot, rest zero); v: [P, heads*dv_slot]."""
    P = q.shape[0]
    o = empty((P, heads * dv_slot), BF16, q)
    lse = empty((n_img, heads, seq), F32, q)
    L.causal_attn_fwd(q, k, v, o, lse, n_img, seq, heads, qk_slot, dv_slot, strict, impl=ATTN_IMPL,
                      dk_true=dk_true)
    return o, lse


def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, n_img, seq, heads, dk_true, qk_slot, dv_slot, strict):
    delta = empty((n_img, heads, seq), F32, q)
    L.causal_attn_bwd(q, k, v, o, do, lse, delta, None, dq, dk, dv, n_img, seq, heads, qk_slot, dv_slot, strict,
                      impl=ATTN_IMPL, dk_true=dk_true)
