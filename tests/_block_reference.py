"""Float64 stage references and element-wise bounds for ImageGPT's fused stack (models/image_gpt.py: the input
convolution, `_block_fwd` / `_block_bwd` per transformer block and the head), written once as a chain of stages.
Shared by tests/test_block_bounds_cpu.py and tests/test_block_kernels_gpu.py through tests/_block_replay.py; not a
test module.

Stage replay.  Worst-case bounds pushed end to end through a block grow by about sqrt(K) per GEMM and say nothing after
two.  So `run` computes every stage from that stage's actual inputs, and each stage is held to its own kernel's bound
(tests/_gemm_reference.py, _attention_reference.py, _step_reference.py, _act_reference.py).  The inputs are chosen by
ROLE, never taken from the arguments the product passed to the kernel call:
  * the cotangent G;
  * the module's fp32 parameters (`weights`): matrices rounded to bf16 by the test, in true heads (head h = channels
    h dk .. (h + 1) dk, `_kv` = all of k, then all of v, as oracle/reference_path.py's causal_attention splits it);
    biases and LayerNorm parameters in fp32; the input convolution with the causal mask applied;
  * the activations the forward saved, and the backward intermediates recorded from earlier stages.
The `mode` object decides what a later stage reads: the kernel's own tensor for the stage (`take` checks it against the
reference first: stage replay), or the reference itself (the float64 chain that tests/test_block_bounds_cpu.py pins to
the oracle's autograd).  A stage fed the wrong tensor, weight, residual, scale or gradient view misses its reference.

Bounds (U24 = 2^-24, U8 = 2^-8; no safety factor except SAFETY = 2 on the attention bounds, as
tests/_attention_reference.py applies it):
  * GEMM, forward and dgrad (`_gemm`): y = A B^T + bias + res_1 + ... with bf16 operands and fp32 sums over the kernel's
    contraction length K (padded slot / stream columns add exact zeros): (K + 1 + n) U24 (|A| |B|^T + |bias| + sum|res|)
    for n added vectors: the recursive-summation chain of tests/_gemm_reference.py with one rounding per epilogue add.
  * A bf16-rounded output (`_round`): b + U8 (|ref| + b), the rounding of the fp32 value, which is within b of ref.
  * du = bf16((dy W2) u): the dgrad bound b times |u| (u is the saved bf16 operand, exact), one fp32 multiply
    U24 (|ref| + |u| b), then `_round`.
  * GELU stage: pre = a2 W1^T + b1 within b_pre.  g = bf16(GELU(pre~)): |GELU'| <= 1.13 moves it by 1.13 b_pre, the
    kernels' GELU fit adds act_err at |pre| + b_pre (its term grows with |x|); then `_round`.  u = bf16(GELU'(pre~)):
    |GELU''| <= 0.80 moves it by 0.80 b_pre, the fit's derivative adds deriv_err; then `_round`.
  * Weight gradients (`_wgrad`): dW = dy^T a over the P pixels, accumulated into the zeroed arena by a split-K launch
    with the split of ops._split_k_for: tests/_gemm_reference.bound(P, 1, |dy|^T |a|, c0 = 0, split).  Their bias
    gradients, reduced from the same tiles: rowsum_bound.
  * LayerNorm forward / backward, the input convolution and column sums: tests/_step_reference.py, the backward from the
    statistics the forward saved and with the residual gradients by role; the bf16 copy of a LayerNorm backward's fp32
    output must be that output rounded, bit for bit (`take_bits`).
  * Attention: tests/_attention_reference.attention on the kernel's q, k, v (and, backward, its recorded do) with the
    scale 1 / sqrt(C / H), whatever slot width the heads live in.
  * dpos = the input convolution's dx summed over the n images: sum_n b_dx + (n + 2) U24 sum_n (|dx| + b_dx).
  * dl = bf16(G) exactly (a zero bound)."""

import math
import re
from typing import NamedTuple

import torch

import _checks
from _act_reference import GELU, act_err, deriv_err
from _attention_reference import SAFETY, attention
from _gemm_reference import bound as gemm_bound
from _gemm_reference import rowsum_bound
from _step_reference import colsum_reference, conv_reference, ln_bwd_reference, ln_fwd_reference

F64, BF16 = torch.float64, torch.bfloat16
U24, U8 = 2.0 ** -24, 2.0 ** -8
GELU1_MAX, GELU2_MAX = 1.13, 0.80  # max |GELU'| (1.129 at x = sqrt 2) and max |GELU''| (0.798 at x = 0)


class Geometry(NamedTuple):
    """Shapes of one run: images n x cin x h x w, C stream channels in H heads of dk, the kernel slot widths and the
    padded stream (c_p) and hidden (f_p) widths of models.image_gpt.StreamLayout."""
    n: int
    cin: int
    h: int
    w: int
    C: int
    H: int
    cout: int
    dk: int
    qk_slot: int
    dv_slot: int
    c_p: int
    f_p: int

    @property
    def S(self):
        return self.h * self.w

    @property
    def P(self):
        return self.n * self.h * self.w

    @property
    def qkv_cols(self):
        return self.H * (2 * self.qk_slot + self.dv_slot)


def geometry(n, cin, h, w, C, H, cout):
    from pytorch_generative_b200 import ops

    dk = C // H
    qs, vs = ops.head_slots(dk, dk)
    return Geometry(n, cin, h, w, C, H, cout, dk, qs, vs, ops.round_up(C, 8), ops.round_up(4 * C, 8))


def kind(name):
    """A stage or gradient name without its block index: 'b1.qkv' -> 'qkv', 'grad _transformer.0._ln1.weight' ->
    'grad _ln1.weight'."""
    return re.sub(r"^b\d+\.|_transformer\.\d+\.", "", name)


# ----------------------------------------------------------------------------------------------------------------------
# weights by role
# ----------------------------------------------------------------------------------------------------------------------
def weights(params, n_blocks, rnd):
    """float64 weights from `params` (parameter name -> tensor, the names of ImageGPT.named_parameters()); rnd rounds a
    weight matrix as the tensor cores read it (bf16, or nothing in the float64 chain)."""
    from oracle.reference_path import causal_mask

    f = lambda k: params[k].detach().to(F64)
    m = lambda k: rnd(params[k].detach()).to(F64).reshape(params[k].shape[0], -1)
    in_w = f("_input.weight")
    W = dict(in_w=in_w * causal_mask(*in_w.shape[2:], True).to(in_w), in_b=f("_input.bias"), pos=f("_pos"),
             ln_w=f("_ln.weight"), ln_b=f("_ln.bias"), wo=m("_out.weight"), bo=f("_out.bias"), blocks=[])
    for b in range(n_blocks):
        p = f"_transformer.{b}."
        kv, bkv = m(p + "_attn._kv.weight"), f(p + "_attn._kv.bias")
        C = kv.shape[1]
        blk = dict(ln1_w=f(p + "_ln1.weight"), ln1_b=f(p + "_ln1.bias"), wq=m(p + "_attn._q.weight"),
                   bq=f(p + "_attn._q.bias"), wk=kv[:C], bk=bkv[:C], wv=kv[C:], bv=bkv[C:],
                   wp=m(p + "_attn._proj.weight"), bp=f(p + "_attn._proj.bias"), ln2_w=f(p + "_ln2.weight"),
                   ln2_b=f(p + "_ln2.bias"), w1=m(p + "_out.0.weight"), b1=f(p + "_out.0.bias"),
                   w2=m(p + "_out.2.weight"), b2=f(p + "_out.2.bias"))
        blk["wqkv"] = torch.cat((blk["wq"], blk["wk"], blk["wv"]))
        blk["bqkv"] = torch.cat((blk["bq"], blk["bk"], blk["bv"]))
        W["blocks"].append(blk)
    return W


# ----------------------------------------------------------------------------------------------------------------------
# stage bounds
# ----------------------------------------------------------------------------------------------------------------------
def _round(ref, b):
    return b + U8 * (ref.abs() + b)


def _gemm(a, w, K, bias=None, res=()):
    """(a w^T + bias + sum res, its fp32 bound) for a contraction of length K."""
    ref, mag, n = a @ w.T, a.abs() @ w.abs().T, 0
    for t in ([bias] if bias is not None else []) + list(res):
        ref, mag, n = ref + t, mag + t.abs(), n + 1
    return ref, (K + 1 + n) * U24 * mag


def _wgrad(dy, a, m_out, n_out, mode):
    """(dy^T a, its bound) as ops.linear_wgrad computes it into a zeroed [m_out, n_out] arena slice."""
    P = dy.shape[0]
    ref = dy.T @ a
    return ref, gemm_bound(P, 1.0, dy.abs().T @ a.abs(), torch.zeros_like(ref), mode.split(m_out, n_out, P))


def _bias_wgrad(dy, m_out, n_out, mode):
    P = dy.shape[0]
    return dy.sum(0), rowsum_bound(P, dy.abs().sum(0), torch.zeros_like(dy[0]), mode.split(m_out, n_out, P))


def _gelu(pre, b_pre):
    """(g, b_g, u, b_u): bf16 GELU(pre) and GELU'(pre) of a pre-activation known within b_pre."""
    g = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
    u = 0.5 * (1 + torch.erf(pre / math.sqrt(2))) + pre * torch.exp(-0.5 * pre * pre) / math.sqrt(2 * math.pi)
    _, a_g = act_err(GELU, pre.abs() + b_pre)
    _, a_u = deriv_err(GELU, pre)
    return g, _round(g, GELU1_MAX * b_pre + a_g), u, _round(u, GELU2_MAX * b_pre + a_u)


def _heads(t, g, d):
    """[P, H d] -> [n, H, S, d]."""
    return t.reshape(g.n, g.S, g.H, d).permute(0, 2, 1, 3)


def _pm(t):
    """[n, H, S, d] -> [P, H d]."""
    n, H, S, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(n * S, H * d)


# ----------------------------------------------------------------------------------------------------------------------
# the stack, stage by stage
# ----------------------------------------------------------------------------------------------------------------------
def run(W, g, x_in, G, eps, mode):
    """Forward and backward of the stack on x_in = x + pos [n, cin, h, w] with cotangent G [P, cout] (pixel-major),
    float64.  Every stage goes through mode.take (activations, intermediates), mode.take_bits (bf16 copies of fp32
    LayerNorm gradients) or mode.grad (parameter gradients, by parameter name).  Returns the logits [P, cout]."""
    C, H, dk, P = g.C, g.H, g.dk, g.P
    kh, kw = W["in_w"].shape[2:]
    pad = (kh // 2, kw // 2)
    cv = conv_reference(x_in, W["in_w"], W["in_b"], torch.zeros(P, C, dtype=F64, device=x_in.device), pad)
    xs = mode.take("stem.xs", cv["out"], cv["b_out"])
    acts = []
    for b, w in enumerate(W["blocks"]):
        s, a = f"b{b}.", {"xs": xs}
        ln = ln_fwd_reference(xs, w["ln1_w"], w["ln1_b"], eps)
        a["mean1"] = mode.take(s + "mean1", ln["mean"], ln["b_mean"])
        a["rstd1"] = mode.take(s + "rstd1", ln["rstd"], ln["b_rstd"])
        a["a1"] = mode.take(s + "a1", ln["y"], _round(ln["y"], ln["b_y"]))
        ref, bd = _gemm(a["a1"], w["wqkv"], g.c_p, bias=w["bqkv"])
        qkv = mode.take(s + "qkv", ref, _round(ref, bd))
        a["q"], a["k"], a["v"] = (_heads(t, g, dk) for t in qkv.split(C, dim=1))
        at = attention(a["q"], a["k"], a["v"], a["v"], False, dk, g.qk_slot, g.dv_slot, backward=False)
        a["o"] = mode.take(s + "o", _pm(at["o"]), SAFETY * _pm(at["b_o"]))
        mode.take(s + "lse", at["lse"], SAFETY * at["b_lse"])
        ref, bd = _gemm(a["o"], w["wp"], H * g.dv_slot, bias=w["bp"], res=(xs,))
        a["h"] = mode.take(s + "h", ref, bd)
        ln = ln_fwd_reference(a["h"], w["ln2_w"], w["ln2_b"], eps)
        a["mean2"] = mode.take(s + "mean2", ln["mean"], ln["b_mean"])
        a["rstd2"] = mode.take(s + "rstd2", ln["rstd"], ln["b_rstd"])
        a["a2"] = mode.take(s + "a2", ln["y"], _round(ln["y"], ln["b_y"]))
        pre, b_pre = _gemm(a["a2"], w["w1"], g.c_p, bias=w["b1"])
        gl, b_g, u, b_u = _gelu(pre, b_pre)
        a["g"], a["u"] = mode.take(s + "g", gl, b_g), mode.take(s + "u", u, b_u)
        ref, bd = _gemm(a["g"], w["w2"], g.f_p, bias=w["b2"], res=(xs, a["h"]))
        acts.append(a)
        xs = mode.take(s + "x_next", ref, bd)
    ln = ln_fwd_reference(xs, W["ln_w"], W["ln_b"], eps)
    mean_f = mode.take("head.mean", ln["mean"], ln["b_mean"])
    rstd_f = mode.take("head.rstd", ln["rstd"], ln["b_rstd"])
    af = mode.take("head.af", ln["y"], _round(ln["y"], ln["b_y"]))
    ref, bd = _gemm(af, W["wo"], g.c_p, bias=W["bo"])
    logits = mode.take("head.logits", ref, bd)

    # head: logits = 1x1(LN(x))
    dl_ref = mode.rnd(G)
    dl = mode.take("head.dl", dl_ref, torch.zeros_like(dl_ref))
    mode.grad("_out.bias", *colsum_reference(dl))
    mode.grad("_out.weight", *_wgrad(dl, af, (g.cout + 7) // 8 * 8, g.c_p, mode))
    ref, bd = _gemm(dl, W["wo"].T, g.cout)
    daf = mode.take("head.daf", ref, _round(ref, bd))
    lb = ln_bwd_reference(daf, xs, W["ln_w"], mean_f, rstd_f)
    dx = mode.take("head.dx", lb["dx"], lb["b_dx"])
    dx_b = mode.take_bits("head.dx_b", dx)
    mode.grad("_ln.weight", lb["dgamma"], lb["b_dgamma"])
    mode.grad("_ln.bias", lb["dbeta"], lb["b_dbeta"])
    dx_sum = (lb["colsum"], lb["b_colsum"])
    for b in reversed(range(len(acts))):
        s, p, a, w = f"b{b}.", f"_transformer.{b}.", acts[b], W["blocks"][b]
        # x_next = x + h + fc2(gelu(fc1(ln2(h)))): fc2's bias gradient is the column sums of the gradient entering
        mode.grad(p + "_out.2.bias", *dx_sum)
        mode.grad(p + "_out.2.weight", *_wgrad(dx_b, a["g"], g.c_p, g.f_p, mode))
        ref, bd = _gemm(dx_b, w["w2"].T, g.c_p)
        du_ref = ref * a["u"]
        b_du = a["u"].abs() * bd + U24 * (du_ref.abs() + a["u"].abs() * bd)
        du = mode.take(s + "du", du_ref, _round(du_ref, b_du))
        mode.grad(p + "_out.0.weight", *_wgrad(du, a["a2"], g.f_p, g.c_p, mode))
        mode.grad(p + "_out.0.bias", *_bias_wgrad(du, g.f_p, g.c_p, mode))
        ref, bd = _gemm(du, w["w1"].T, g.f_p)
        da2 = mode.take(s + "da2", ref, _round(ref, bd))
        # h receives LN2's backward and the direct gradient of x_next
        lb = ln_bwd_reference(da2, a["h"], w["ln2_w"], a["mean2"], a["rstd2"], dres0=dx)
        dh = mode.take(s + "dh", lb["dx"], lb["b_dx"])
        dh_b = mode.take_bits(s + "dh_b", dh)
        mode.grad(p + "_ln2.weight", lb["dgamma"], lb["b_dgamma"])
        mode.grad(p + "_ln2.bias", lb["dbeta"], lb["b_dbeta"])
        mode.grad(p + "_attn._proj.bias", lb["colsum"], lb["b_colsum"])
        # h = x + proj(attention(ln1(x)))
        mode.grad(p + "_attn._proj.weight", *_wgrad(dh_b, a["o"], g.c_p, H * g.dv_slot, mode))
        ref, bd = _gemm(dh_b, w["wp"].T, g.c_p)
        do = mode.take(s + "do", ref, _round(ref, bd))
        at = attention(a["q"], a["k"], a["v"], _heads(do, g, dk), False, dk, g.qk_slot, g.dv_slot)
        dq = mode.take(s + "dq", _pm(at["dq"]), SAFETY * _pm(at["b_dq"]))
        dk_ = mode.take(s + "dk", _pm(at["dk"]), SAFETY * _pm(at["b_dk"]))
        dv = mode.take(s + "dv", _pm(at["dv"]), SAFETY * _pm(at["b_dv"]))
        dqkv = torch.cat((dq, dk_, dv), dim=1)
        ref, bd = _wgrad(dqkv, a["a1"], g.qkv_cols, g.c_p, mode)
        mode.grad(p + "_attn._q.weight", ref[:C], bd[:C])
        mode.grad(p + "_attn._kv.weight", ref[C:], bd[C:])
        ref, bd = _bias_wgrad(dqkv, g.qkv_cols, g.c_p, mode)
        mode.grad(p + "_attn._q.bias", ref[:C], bd[:C])
        mode.grad(p + "_attn._kv.bias", ref[C:], bd[C:])
        ref, bd = _gemm(dqkv, w["wqkv"].T, g.qkv_cols)
        da1 = mode.take(s + "da1", ref, _round(ref, bd))
        # x receives LN1's backward, the direct gradient of h and that of x_next
        lb = ln_bwd_reference(da1, a["xs"], w["ln1_w"], a["mean1"], a["rstd1"], dres0=dx, dres1=dh)
        dx = mode.take(s + "dx_in", lb["dx"], lb["b_dx"])
        dx_b = mode.take_bits(s + "dx_in_b", dx)
        mode.grad(p + "_ln1.weight", lb["dgamma"], lb["b_dgamma"])
        mode.grad(p + "_ln1.bias", lb["dbeta"], lb["b_dbeta"])
        dx_sum = (lb["colsum"], lb["b_colsum"])

    # stem: x = conv(x_img + pos); its bias gradient is the column sums of the gradient entering block 0
    mode.grad("_input.bias", *dx_sum)
    dx = mode.take("stem.dy", dx, torch.zeros_like(dx))
    cv = conv_reference(x_in, W["in_w"], W["in_b"], dx, pad)
    mode.grad("_input.weight", cv["dw"], cv["b_dw"])
    n, _, h, wd = x_in.shape
    dpos, b_dpos = torch.zeros_like(W["pos"]), torch.zeros_like(W["pos"])
    dpos[:, :, :h, :wd] = cv["dx"].sum(0, keepdim=True)
    b_dpos[:, :, :h, :wd] = (cv["b_dx"].sum(0) + (n + 2) * U24 * (cv["dx"].abs() + cv["b_dx"]).sum(0))[None]
    mode.grad("_pos", dpos, b_dpos)
    return logits


# ----------------------------------------------------------------------------------------------------------------------
# modes
# ----------------------------------------------------------------------------------------------------------------------
class Chain:
    """The float64 chain: every stage reads the reference of the stages before it; gradients are collected by name."""

    def __init__(self):
        self.grads = {}

    def take(self, name, ref, bound):
        return ref

    def take_bits(self, name, x):
        return x

    def grad(self, name, ref, bound):
        self.grads[name] = ref

    def split(self, m_out, n_out, k):
        return 1

    @staticmethod
    def rnd(t):
        return t.to(F64)


class Replay:
    """Stage replay against the kernels: `kernel` maps each stage name to the tensor the product computed for it, in
    true-head, unpadded layout; `params` maps parameter names to the module's parameters (their .grad is checked).
    Failures are collected per stage (`failures`), the worst |err| / bound per stage in `ratios`."""

    def __init__(self, kernel, params):
        self.kernel, self.params = kernel, params
        self.ratios, self.failures = {}, {}

    def _check(self, name, got, ref, bound):
        err = (got.to(F64) - ref).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound).nan_to_num(nan=math.inf)
        self.ratios[name] = float(ratio.max()) if ratio.numel() else 0.0
        try:
            _checks.check(name, got, ref, bound)
        except AssertionError as e:
            self.failures[name] = str(e)

    def take(self, name, ref, bound):
        got = self.kernel[name]
        self._check(name, got, ref, bound)
        return got.to(F64)

    def take_bits(self, name, x):
        got = self.kernel[name]
        try:
            _checks.check_equal(name, got, x.to(got.dtype))
            self.ratios[name] = 0.0
        except AssertionError as e:
            self.failures[name] = str(e)
            self.ratios[name] = math.inf
        return got.to(F64)

    def grad(self, name, ref, bound):
        got = self.params[name].grad
        if got is None:
            self.failures["grad " + name] = "no gradient"
            return
        self._check("grad " + name, got, ref.reshape(got.shape), bound.reshape(got.shape))

    def zero(self, name, t):
        """Pad columns / rows that must hold exact zeros."""
        if t.numel() and t.any():
            self.failures[name] = f"{name}: {int((t != 0).sum())} nonzero elements"

    def split(self, m_out, n_out, k):
        from pytorch_generative_b200 import ops

        return ops._split_k_for(m_out, n_out, k)

    @staticmethod
    def rnd(t):
        return t.to(BF16).to(F64)

    def failed_kinds(self):
        return sorted({kind(n) for n in self.failures})

    def worst_by_kind(self):
        out = {}
        for n, r in self.ratios.items():
            out[kind(n)] = max(out.get(kind(n), 0.0), r)
        return out
