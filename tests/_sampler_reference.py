"""The per-pixel programs of the incremental sampler (models/incremental.py; `_pixel_program` of PixelCNN,
GatedPixelCNN, PixelSNAIL and ImageGPT) as a stage graph, float64 references of every stage kind, their element-wise
bounds and `chain`, which composes the references along the graph.  Shared by tests/test_sampler_bounds_cpu.py and
tests/test_sampler_stages_gpu.py (through tests/_sampler_replay.py); not a test module.

Stage graph.  `graph(model, state, shape, n_heads)` reads the program from a state dict along
oracle/reference_path.py, never from the product's tap tables (`live_taps`, `PixelStepper.table`) or its packing
(`_pack_pixel_weights`, `incremental.pack`), so a wrong table or a wrong packing fails.  A stage evaluates one position
p of every image.  It names
  * its kind: `linear` (a GEMM of the skinny or tensor-core kernel with its bias / residual / activation epilogue),
    `act` (act_cast), `gate` (pm.gated, tanh), `gated_res` (pm.gated_res, identity gate), `decode` (pg_attn_decode),
    `ln` (a single-row LayerNorm), `conv_small` (ImageGPT's input convolution on the window around p), or a `virtual`
    step no kernel records (an fp32 sum, GatedPixelCNN's row mask, the window's centre row): the graph computes it and
    its consumers are held to it;
  * its operand (`src`) and residuals (`res`) as sources: the output of an earlier stage of the same step, or a gather
    of cache rows at tap offsets that come from `causal_mask`, the kernel sizes and the paddings (a tap outside the
    image reads zeros), or a cache row of the previous pixel (the fix-ups), or the final canvas;
  * the layouts of its operand and output: the column of every true channel in the padded pitch (`padded`, a gate's
    halves each at its own pitch), the attention head slots (`slots`), tap-major gathers; every other column is a pad
    column and holds +0.0;
  * which cache it writes (`CacheSpec`): row p at step p, or row p - 1 at step p for the fix-ups (lag 1).

References and bounds (U24 = 2^-24, U8 = 2^-8 the unit roundoffs of fp32 and bf16).  Every reference is computed in
float64 from the stage's recorded inputs and the state dict's weights (masked, rounded to bf16 as the kernels read
them) and fp32 biases:
  * linear: y = a W^T + b + res0 + res1 with K = the operand's padded width: the fp32 chain of tests/_gemm_reference.py
    (K + 1) U24 plus one U24 for the bias and for each residual, times |a| |W|^T + |b| + sum |res|.  A bf16 output adds
    U8 of itself; ReLU is 1-Lipschitz; ELU and GELU add tests/_act_reference.act_err (GELU's slope is below 1.13);
  * act: ReLU and the identity are exact before the bf16 rounding (bit for bit); ELU within act_err and one rounding;
  * gate / gated_res: tests/_act_reference.gate_fwd_err, one bf16 rounding / one fp32 add;
  * decode: tests/_attention_reference.decode_row over cache rows <= p (< p when strict), with that module's SAFETY;
  * ln: tests/_step_reference.ln_fwd_reference, one bf16 rounding;
  * conv_small: tests/_step_reference.conv_reference on the recorded window.
No bound is loosened for the sampler: these are the training path's bounds applied to one row per image."""

import collections
import math

import torch
import torch.nn.functional as F

from _act_reference import ELU, GELU, NONE, RELU, TANH, act64, act_err, gate_fwd_err, gate_ref
from _attention_reference import SAFETY, decode_row
from _step_reference import conv_reference, ln_fwd_reference
from oracle.reference_path import _count, causal_mask, image_positional_encoding

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U24, U8 = 2.0 ** -24, 2.0 ** -8
SLOTS = (64, 128)  # the attention kernels' head-slot widths (pg_attention.cu)
GELU_SLOPE = 1.13  # max |GELU'| = 1.1289


def round_up(v, m):
    return (v + m - 1) // m * m


# ----------------------------------------------------------------------------------------------------------------------
# layouts
# ----------------------------------------------------------------------------------------------------------------------
Layout = collections.namedtuple("Layout", "cols width")  # the column of each true channel; the row width


def padded(C, parts=1):
    """C channels made of `parts` equal parts, each part at the 16-byte operand pitch (round_up(part, 8) columns)."""
    part = C // parts
    step = round_up(part, 8)
    return Layout([g * step + i for g in range(parts) for i in range(part)], parts * step)


def exact(C):
    return Layout(list(range(C)), C)


def slots(H, d, slot, base=0, width=None):
    return Layout([base + h * slot + i for h in range(H) for i in range(d)], width or base + H * slot)


def tapmajor(lay, T):
    return Layout([t * lay.width + c for t in range(T) for c in lay.cols], T * lay.width)


def cat(*lays):
    cols, off = [], 0
    for lay in lays:
        cols += [off + c for c in lay.cols]
        off += lay.width
    return Layout(cols, off)


def pad_cols(lay):
    keep = set(lay.cols)
    return [c for c in range(lay.width) if c not in keep]


def slot(d):
    return next(s for s in SLOTS if d <= s)


# ----------------------------------------------------------------------------------------------------------------------
# the stage graph
# ----------------------------------------------------------------------------------------------------------------------
class Stage:
    """One step of a per-pixel program (see the module docstring).  w64: [Cout, T * Cin] float64 of the bf16 weight,
    tap-major like the operand's true channels; b64 the bias; lay_in / lay_out the operand's and output's layouts."""

    def __init__(self, name, kind, src=None, res=(), w=None, b=None, act=NONE, f32=False, lay_in=None, lay_out=None,
                 writes=(), pads=True, w_bf16=True, **extra):
        self.name, self.kind, self.src, self.res = name, kind, src, tuple(res)
        self.w64 = None if w is None else (w.detach().to(BF16) if w_bf16 else w.detach()).to(F64)
        self.wx = None if w is None else w.detach().to(F64)  # the state dict's value: the chain's weight
        self.b64 = None if b is None else b.detach().to(F64)
        self.act, self.f32, self.lay_in, self.lay_out = act, f32, lay_in, lay_out
        self.writes, self.pads = tuple(writes), pads
        self.__dict__.update(extra)


CacheSpec = collections.namedtuple("CacheSpec", "writer which lo hi lag layout")  # row r = writer's output at step r + lag


class Graph:
    def __init__(self, model, n, c, h, w):
        self.model, self.n, self.c, self.h, self.w, self.S = model, n, c, h, w, h * w
        self.stages, self.stage, self.caches = [], {}, {}
        self.caches["image"] = CacheSpec(None, None, 0, c, 0, padded(c))

    def add(self, *a, **kw):
        s = Stage(*a, **kw)
        self.stages.append(s)
        self.stage[s.name] = s
        return s

    def recorded(self):
        return [s for s in self.stages if s.kind != "virtual"]


def _taps(weight, mask=None):
    """[(i, j)] of the live kernel positions, row-major like the weight."""
    kh, kw = weight.shape[-2:]
    m = torch.ones(kh, kw) if mask is None else mask
    return [(i, j) for i in range(kh) for j in range(kw) if float(m[i, j]) != 0.0]


def _wmat(weight, taps, mask=None):
    """[Cout, T * Cin]: the weight (times the causal mask) at the kernel positions `taps`, tap-major."""
    w = weight.detach() if mask is None else weight.detach() * mask.to(weight.dtype)
    return torch.stack([w[:, :, i, j] for i, j in taps], 1).reshape(w.shape[0], -1)


def _conv_stage(G, name, state, key, src, taps, lay_in, lay_out, mask=None, **kw):
    return G.add(name, "linear", src, w=_wmat(state[key + ".weight"], taps, mask), b=state[key + ".bias"],
                 lay_in=lay_in, lay_out=lay_out, **kw)


def _gather(cache, offsets):
    return ("gather", cache, tuple(offsets))


def pixel_cnn(state, n, c, h, w):
    G = Graph("pixel_cnn", n, c, h, w)
    win = state["_input.weight"]
    R2, kh, kw = win.shape[0], win.shape[2], win.shape[3]
    half = state["_causal_layers.0._net.1.weight"].shape[0] if _count(state, "_causal_layers") else R2 // 2
    m_in = causal_mask(kh, kw, True)
    t_in = _taps(win, m_in)
    _conv_stage(G, "in", state, "_input", _gather("image", [(i - kh // 2, j - kw // 2) for i, j in t_in]), t_in,
                tapmajor(padded(c), len(t_in)), padded(R2), mask=m_in, f32=True)
    x = "in"
    for i in range(_count(state, "_causal_layers")):
        pre = f"_causal_layers.{i}._net."
        m3 = causal_mask(3, 3, False)
        t3 = _taps(state[pre + "3.weight"], m3)
        G.caches[f"t1.{i}"] = CacheSpec(f"b{i}_1", "b", 0, half, 0, padded(half))
        G.add(f"b{i}_act", "act", ("value", x), act=RELU, lay_in=padded(R2), lay_out=padded(R2))
        _conv_stage(G, f"b{i}_1", state, pre + "1", ("value", f"b{i}_act"), [(0, 0)], padded(R2), padded(half),
                    act=RELU, writes=(f"t1.{i}",))
        _conv_stage(G, f"b{i}_3", state, pre + "3", _gather(f"t1.{i}", [(a - 1, b - 1) for a, b in t3]), t3,
                    tapmajor(padded(half), len(t3)), padded(half), mask=m3, act=RELU)
        _conv_stage(G, f"b{i}_5", state, pre + "5", ("value", f"b{i}_3"), [(0, 0)], padded(half), padded(R2),
                    res=(("value", x), ("value", x)), f32=True)
        x = f"b{i}_5"
    hc, cout = state["_head.1.weight"].shape[0], state["_head.3.weight"].shape[0]
    G.add("h_act", "act", ("value", x), act=RELU, lay_in=padded(R2), lay_out=padded(R2))
    _conv_stage(G, "h1", state, "_head.1", ("value", "h_act"), [(0, 0)], padded(R2), padded(hc), act=RELU)
    _conv_stage(G, "logits", state, "_head.3", ("value", "h1"), [(0, 0)], padded(hc), exact(cout), f32=True)
    return G


def gated_pixel_cnn(state, n, c, h, w):
    G = Graph("gated_pixel_cnn", n, c, h, w)
    pres = ["_input"] + [f"_gated_layers.{i}" for i in range(_count(state, "_gated_layers"))]
    C = state["_input._vstack_1xN.weight"].shape[0]
    last = len(pres) - 1
    pC, p2 = padded(C), padded(2 * C, 2)
    # (1) the previous pixel is final: finish its vertical-stack outputs (row p - 1; at p = 0 a row that p = 1 redoes)
    for i in range(last):
        pre = pres[i]
        src = ("row", "image", 1) if i == 0 else ("value", f"fv{i - 1}")
        G.caches[f"vc.{i}"] = CacheSpec(f"fv{i}", "b", 0, C, 1, pC)
        _conv_stage(G, f"vx{i}", state, pre + "._vstack_1x1", src, [(0, 0)], padded(c) if i == 0 else pC, p2,
                    res=(("prev", f"v2_{i}"),), fixup=True)
        G.add(f"fv{i}", "gate", ("value", f"vx{i}"), lay_in=p2, lay_out=pC, writes=(f"vc.{i}",), fixup=True)
    # (2) position p
    for i, pre in enumerate(pres):
        k = state[pre + "._vstack_1xN.weight"].shape[-1]
        p = (k - 1) // 2
        causal = i == 0
        r = k // 2 + 1
        cin, lin = (c, padded(c)) if causal else (C, pC)
        vsrc, hsrc = ("image", "image") if causal else (f"vc.{i - 1}", f"hc.{i - 1}")
        # the 1xN rows the (k // 2 + 1) x 1 convolution reads: rows y + ii - p - 1 (padding p + 1, front crop)
        offs = [(ii - p - 1, j - p) for ii in range(r) for j in range(k)]
        _conv_stage(G, f"v1_{i}", state, pre + "._vstack_1xN", ("rows", _gather(vsrc, offs), r),
                    [(0, j) for j in range(k)], tapmajor(lin, k), pC)
        G.add(f"v1m_{i}", "virtual", ("valid", ("value", f"v1_{i}"), r, p), lay_out=pC)
        _conv_stage(G, f"v2_{i}", state, pre + "._vstack_Nx1", ("value", f"v1m_{i}"), [(ii, 0) for ii in range(r)],
                    tapmajor(pC, r), p2)
        _conv_stage(G, f"ln{i}", state, pre + "._link", ("value", f"v2_{i}"), [(0, 0)], p2, p2)
        mc = int(causal)
        _conv_stage(G, f"h{i}", state, pre + "._hstack_1xN", _gather(hsrc, [(0, j - p - mc) for j in range(r)]),
                    [(0, j) for j in range(r)], tapmajor(lin, r), p2, res=(("value", f"ln{i}"),))
        G.add(f"g{i}", "gate", ("value", f"h{i}"), lay_in=p2, lay_out=pC)
        _conv_stage(G, f"hs{i}", state, pre + "._hstack_skip", ("value", f"g{i}"), [(0, 0)], pC, pC,
                    res=() if causal else (("value", f"hs{i - 1}"),), f32=True)
        if i < last:
            G.caches[f"hc.{i}"] = CacheSpec(f"hr{i}", "b", 0, C, 0, pC)
        _conv_stage(G, f"hr{i}", state, pre + "._hstack_residual", ("value", f"g{i}"), [(0, 0)], pC, pC,
                    res=() if causal else (("value", f"hr{i - 1}"),), f32=True, both=True,
                    writes=(f"hc.{i}",) if i < last else ())
    hc, cout = state["_head.1.weight"].shape[0], state["_head.3.weight"].shape[0]
    G.add("h_act", "act", ("value", f"hs{last}"), act=RELU, lay_in=pC, lay_out=pC)
    _conv_stage(G, "h1", state, "_head.1", ("value", "h_act"), [(0, 0)], pC, padded(hc), act=RELU)
    _conv_stage(G, "logits", state, "_head.3", ("value", "h1"), [(0, 0)], padded(hc), exact(cout), f32=True)
    return G


def pixel_snail(state, n, c, h, w):
    G = Graph("pixel_snail", n, c, h, w)
    win = state["_input.weight"]
    C = win.shape[0]
    pC, p2 = padded(C), padded(2 * C, 2)
    blocks = [f"_pixel_snail_blocks.{i}" for i in range(_count(state, "_pixel_snail_blocks"))]
    t22 = [(0, 0), (0, 1), (1, 0), (1, 1)]
    off22 = [(i - 1, j - 1) for i, j in t22]  # 2x2, padding 1, front crop
    ckv = round_up(2 + C + c, 8)
    kv_in = Layout(list(range(2 + C + c)), ckv)
    q_in = Layout(list(range(2 + C)), round_up(C + 2, 8))  # its pad columns may hold image values: the weight ignores them
    att = {}
    for bi, blk in enumerate(blocks):
        key = state[blk + "._attention._q.weight"].shape[0]
        val = state[blk + "._attention._proj.weight"].shape[0]
        qs, vs = slot(key), slot(val)
        att[bi] = (key, val, qs, vs)
        kv_out = cat(slots(1, key, qs), slots(1, val, vs))
        G.caches[f"kc.{bi}"] = CacheSpec(f"kvf{bi}", "b", 0, key, 1, slots(1, key, qs))
        G.caches[f"vc.{bi}"] = CacheSpec(f"kvf{bi}", "b", key, key + val, 1, slots(1, val, vs))
        # (1) the previous pixel's key / value, from its features and its final image value
        src = ("cat", ("prev_akv", bi), ("bf16", ("row", "image", 1)))
        _conv_stage(G, f"kvf{bi}", state, blk + "._attention._kv", src, [(0, 0)], kv_in, kv_out,
                    writes=(f"kc.{bi}", f"vc.{bi}"), fixup=True)
    m_in = causal_mask(*win.shape[2:], True)
    t_in = _taps(win, m_in)
    kh, kw = win.shape[2:]
    _conv_stage(G, "in", state, "_input", _gather("image", [(i - kh // 2, j - kw // 2) for i, j in t_in]), t_in,
                tapmajor(padded(c), len(t_in)), pC, mask=m_in, f32=True)
    x = "in"
    for bi, blk in enumerate(blocks):
        key, val, qs, vs = att[bi]
        res = x
        for j in range(_count(state, blk + "._residual")):
            pre = f"{blk}._residual.{j}"
            G.caches[f"ea.{bi}.{j}"] = CacheSpec(f"ea{bi}_{j}", "b", 0, C, 0, pC)
            G.caches[f"eb.{bi}.{j}"] = CacheSpec(f"ri{bi}_{j}", "b", 0, C, 0, pC)
            G.add(f"ea{bi}_{j}", "act", ("value", res), act=ELU, lay_in=pC, lay_out=pC, writes=(f"ea.{bi}.{j}",))
            _conv_stage(G, f"ri{bi}_{j}", state, pre + "._input_conv", _gather(f"ea.{bi}.{j}", off22), t22,
                        tapmajor(pC, 4), pC, act=ELU, writes=(f"eb.{bi}.{j}",))
            _conv_stage(G, f"ro{bi}_{j}", state, pre + "._output_conv", _gather(f"eb.{bi}.{j}", off22), t22,
                        tapmajor(pC, 4), p2)
            G.add(f"gr{bi}_{j}", "gated_res", ("value", f"ro{bi}_{j}"), res=(("value", res),), lay_in=p2, lay_out=pC,
                  f32=True)
            res = f"gr{bi}_{j}"
        # [position | features | image placeholder (row p is not drawn yet: zero) | 0-pad]
        akv = ("cat", ("bf16", ("pos",)), ("bf16", ("value", res)), ("zeros", c))
        G.add(f"akv{bi}", "virtual", akv, lay_out=kv_in, C=C)
        _conv_stage(G, f"q{bi}", state, blk + "._attention._q", ("slice", ("value", f"akv{bi}"), 0, 2 + C), [(0, 0)], q_in,
                    slots(1, key, qs), pads=False)
        _conv_stage(G, f"kv{bi}", state, blk + "._attention._kv", ("value", f"akv{bi}"), [(0, 0)], kv_in,
                    cat(slots(1, key, qs), slots(1, val, vs)))
        G.add(f"at{bi}", "decode", ("value", f"q{bi}"), kv=f"kv{bi}", kc=f"kc.{bi}", vc=f"vc.{bi}", H=1, dk=key,
              dv=val, qs=qs, vs=vs, strict=True, lay_out=slots(1, val, vs))
        _conv_stage(G, f"pj{bi}", state, blk + "._attention._proj", ("value", f"at{bi}"), [(0, 0)], slots(1, val, vs),
                    padded(val), f32=True)
        G.add(f"rea{bi}", "act", ("value", res), act=ELU, lay_in=pC, lay_out=pC)
        _conv_stage(G, f"rro{bi}", state, blk + "._residual_out", ("value", f"rea{bi}"), [(0, 0)], pC, pC, act=ELU)
        G.add(f"aea{bi}", "act", ("value", f"pj{bi}"), act=ELU, lay_in=padded(val), lay_out=padded(val))
        _conv_stage(G, f"aao{bi}", state, blk + "._attention_out", ("value", f"aea{bi}"), [(0, 0)], padded(val), pC,
                    act=ELU)
        G.add(f"sum{bi}", "virtual", ("f32sum", ("value", f"rro{bi}"), ("value", f"aao{bi}")), lay_out=pC)
        G.add(f"oea{bi}", "act", ("value", f"sum{bi}"), act=ELU, lay_in=pC, lay_out=pC)
        _conv_stage(G, f"out{bi}", state, blk + "._out", ("value", f"oea{bi}"), [(0, 0)], pC, pC, act=ELU)
        G.add(f"x{bi}", "virtual", ("f32sum", ("value", x), ("value", f"out{bi}")), lay_out=pC)
        x = f"x{bi}"
    h2, cout = state["_output.0.weight"].shape[0], state["_output.1.weight"].shape[0]
    _conv_stage(G, "o0", state, "_output.0", ("bf16", ("value", x)), [(0, 0)], pC, padded(h2))
    _conv_stage(G, "logits", state, "_output.1", ("value", "o0"), [(0, 0)], padded(h2), exact(cout), f32=True)
    return G


def image_gpt(state, n, c, h, w, n_heads):
    G = Graph("image_gpt", n, c, h, w)
    win = state["_input.weight"]
    C, kh, kw = win.shape[0], win.shape[2], win.shape[3]
    H, d = n_heads, C // n_heads
    sl = slot(d)
    pC, pF = padded(C), padded(4 * C)
    G.add("conv", "conv_small", ("patch",), w=win.detach() * causal_mask(kh, kw, True), b=state["_input.bias"], kh=kh,
          kw=kw, lay_out=pC, mask=causal_mask(kh, kw, True), w_bf16=False)
    G.add("x_in", "virtual", ("centre", "conv"), lay_out=pC)
    x = "x_in"
    for b in range(_count(state, "_transformer")):
        pre = f"_transformer.{b}."
        G.add(f"ln1_{b}", "ln", ("value", x), g=state[pre + "_ln1.weight"], be=state[pre + "_ln1.bias"], lay_in=pC,
              lay_out=pC)
        wqkv = torch.cat((state[pre + "_attn._q.weight"], state[pre + "_attn._kv.weight"]))
        bqkv = torch.cat((state[pre + "_attn._q.bias"], state[pre + "_attn._kv.bias"]))
        qkv_out = slots(3 * H, d, sl)
        G.add(f"qkv{b}", "linear", ("value", f"ln1_{b}"), w=wqkv.reshape(3 * C, C), b=bqkv, lay_in=pC, lay_out=qkv_out)
        G.caches[f"kc.{b}"] = CacheSpec(f"qkv{b}", "b", C, 2 * C, 0, slots(H, d, sl))
        G.caches[f"vc.{b}"] = CacheSpec(f"qkv{b}", "b", 2 * C, 3 * C, 0, slots(H, d, sl))
        G.add(f"at{b}", "decode", ("value", f"qkv{b}"), kv=f"qkv{b}", kc=f"kc.{b}", vc=f"vc.{b}", H=H, dk=d, dv=d,
              qs=sl, vs=sl, strict=False, lay_out=slots(H, d, sl))
        G.add(f"pj{b}", "linear", ("value", f"at{b}"), res=(("value", x),), w=state[pre + "_attn._proj.weight"].reshape(C, C),
              b=state[pre + "_attn._proj.bias"], lay_in=slots(H, d, sl), lay_out=pC, f32=True)
        G.add(f"ln2_{b}", "ln", ("value", f"pj{b}"), g=state[pre + "_ln2.weight"], be=state[pre + "_ln2.bias"],
              lay_in=pC, lay_out=pC)
        G.add(f"fc1_{b}", "linear", ("value", f"ln2_{b}"), w=state[pre + "_out.0.weight"].reshape(4 * C, C),
              b=state[pre + "_out.0.bias"], act=GELU, lay_in=pC, lay_out=pF)
        G.add(f"fc2_{b}", "linear", ("value", f"fc1_{b}"), res=(("value", x), ("value", f"pj{b}")),
              w=state[pre + "_out.2.weight"].reshape(C, 4 * C), b=state[pre + "_out.2.bias"], lay_in=pF, lay_out=pC,
              f32=True)
        x = f"fc2_{b}"
    G.add("lnf", "ln", ("value", x), g=state["_ln.weight"], be=state["_ln.bias"], lay_in=pC, lay_out=pC)
    cout = state["_out.weight"].shape[0]
    G.add("logits", "linear", ("value", "lnf"), w=state["_out.weight"].reshape(cout, C), b=state["_out.bias"],
          lay_in=pC, lay_out=exact(cout), f32=True)
    G.pos = state["_pos"].detach()
    return G


def graph(model, state, shape, n_heads=None):
    n, c, h, w = shape
    if model == "image_gpt":
        return image_gpt(state, n, c, h, w, n_heads)
    return {"pixel_cnn": pixel_cnn, "gated_pixel_cnn": gated_pixel_cnn, "pixel_snail": pixel_snail}[model](
        state, n, c, h, w)


# ----------------------------------------------------------------------------------------------------------------------
# sources: the values a stage's operand and residuals are made of
# ----------------------------------------------------------------------------------------------------------------------
class Env:
    """The values of a graph's stages at every step, true channels only, [rows, C] float64: computed in float64
    (`exact=True`, the chain) or the product's recorded values (the replay, where `round` applies the product's casts).
    `canvas` is the final canvas; cache rows come from their writer's value at its write step."""

    def __init__(self, G, canvas, exact):
        self.G, self.canvas, self.exact = G, canvas, exact
        self.vals = [dict() for _ in range(G.S)]  # step -> stage -> {"f": value, "b": bf16 value}
        self.S, self.n = G.S, canvas.shape[0]
        self.pos = image_positional_encoding((1, 2, G.h, G.w))[0].reshape(2, -1).t()  # [S, 2] as the oracle's

    def round(self, t):
        return t if self.exact else t.to(F32).to(BF16).to(F64)

    def value(self, p, name, which=None):
        """A stage's value at step p: `which` "f" (fp32 output) or "b" (bf16 output); by default the one its consumers
        read (fp32 for an fp32 stage)."""
        v = self.vals[p][name]
        if which is None:
            which = "f" if "f" in v and (self.G.stage[name].f32 or "b" not in v) else "b"
        return v[which]

    def image(self, r):
        """The final canvas value of pixel r, [n, c]."""
        y, x = divmod(r, self.G.w)
        return self.canvas[:, :, y, x].to(F64)

    def cache_row(self, name, r):
        spec = self.G.caches[name]
        if spec.writer is None:
            return self.round(self.image(r))
        return self.value(r + spec.lag, spec.writer, spec.which)[:, spec.lo:spec.hi]

    def cache_width(self, name):
        spec = self.G.caches[name]
        return spec.hi - spec.lo

    def rows_of(self, p, offsets):
        y, x = divmod(p, self.G.w)
        out = []
        for dy, dx in offsets:
            yy, xx = y + dy, x + dx
            out.append(yy * self.G.w + xx if 0 <= yy < self.G.h and 0 <= xx < self.G.w else None)
        return out

    def ev(self, spec, p):
        kind = spec[0]
        if kind == "value":
            return self.value(p, spec[1])
        if kind == "bf16":
            return self.round(self.ev(spec[1], p))
        if kind == "gather":
            cw = self.cache_width(spec[1])
            parts = [torch.zeros(self.n, cw, dtype=F64) if r is None else self.cache_row(spec[1], r).cpu()
                     for r in self.rows_of(p, spec[2])]
            return torch.cat(parts, 1)
        if kind == "rows":  # a gather of r row-taps, one operand row per (image, row-tap)
            a = self.ev(spec[1], p)
            return a.reshape(self.n * spec[2], -1)
        if kind == "valid":  # GatedPixelCNN: 1xN rows above the image are the Nx1 convolution's zero padding
            v = self.ev(spec[1], p)
            r_taps, pad = spec[2], spec[3]
            y = p // self.G.w
            keep = torch.tensor([float(y + ii - pad - 1 >= 0) for ii in range(r_taps)], dtype=F64)
            return (v.reshape(self.n, r_taps, -1) * keep.view(1, -1, 1)).reshape(self.n, -1)
        if kind == "row":  # a cache row of pixel p - lag (the fix-ups; p = 0 reads row 0)
            return self.cache_row(spec[1], max(p - spec[2], 0))
        if kind == "prev":  # a stage's value at step p - 1 (zero at p = 0: the program's buffers start zeroed)
            if p == 0:
                return torch.zeros(self.n, self.G.stage[spec[1]].w64.shape[0], dtype=F64)
            return self.value(p - 1, spec[1])
        if kind == "prev_akv":  # the attention operand of p - 1 without its image columns: [position | features]
            C = self.G.stage[f"akv{spec[1]}"].C
            if p == 0:  # the operand buffer starts zeroed
                return torch.zeros(self.n, 2 + C, dtype=F64)
            return self.value(p - 1, f"akv{spec[1]}")[:, : 2 + C]
        if kind == "pos":
            return self.pos[p].to(F64).view(1, 2).expand(self.n, 2)
        if kind == "slice":
            return self.ev(spec[1], p)[:, spec[2]:spec[3]]
        if kind == "zeros":
            return torch.zeros(self.n, spec[1], dtype=F64)
        if kind == "cat":
            return torch.cat([self.ev(s, p).cpu() for s in spec[1:]], 1)
        if kind == "f32sum":
            a, b = self.ev(spec[1], p), self.ev(spec[2], p)
            return a + b if self.exact else (a.to(F32) + b.to(F32)).to(F64)
        if kind == "centre":
            st = self.G.stage[spec[1]]
            v = self.value(p, spec[1])
            return v.reshape(self.n, st.kh * st.kw, -1)[:, (st.kh // 2) * st.kw + st.kw // 2]
        if kind == "patch":
            return self.patch(p)
        raise AssertionError(spec)

    def patch(self, p):
        """ImageGPT: [n, c, kh, kw] window of x + pos around p (fp32 sums in the replay, float64 in the chain), zero
        outside the image; the window's pixels at and after p hold the final canvas too (the mask hides them)."""
        st = self.G.stage["conv"]
        y, x = divmod(p, self.G.w)
        out = torch.zeros(self.n, self.G.c, st.kh, st.kw, dtype=F64)
        for i in range(st.kh):
            for j in range(st.kw):
                yy, xx = y + i - st.kh // 2, x + j - st.kw // 2
                if 0 <= yy < self.G.h and 0 <= xx < self.G.w:
                    v, pe = self.canvas[:, :, yy, xx], self.G.pos[0, :, yy, xx].cpu()
                    out[:, :, i, j] = (v.to(F64) + pe.to(F64)) if self.exact else (v.float().cpu() + pe.float()).to(F64)
        return out


# ----------------------------------------------------------------------------------------------------------------------
# float64 references of the stage kinds
# ----------------------------------------------------------------------------------------------------------------------
def linear_ref(st, a, res):
    """(y, its bound before the output's own rounding / activation) from the operand's true channels a [rows, K_true]
    and the residuals' true channels; K is the operand's padded width."""
    w = st.w64.to(a.device)
    b = st.b64.to(a.device)
    y = a @ w.T + b
    mag = a.abs() @ w.abs().T + b.abs()
    for r in res:
        y, mag = y + r, mag + r.abs()
    return y, mag


def linear_bound(st, K, y, mag):
    """{"f": fp32 output bound, "b": bf16 output's reference and bound} of a linear stage."""
    err = (K + 2 + len(st.res)) * U24 * mag
    out = {"f": (y, err)}
    if st.act == NONE:
        out["b"] = (y, err * (1 + U8) + U8 * y.abs())
    elif st.act == RELU:
        r = y.clamp_min(0)
        out["b"] = (r, err * (1 + U8) + U8 * r.abs())
    elif st.act == ELU:
        e = act64(ELU, y)
        rr, _ = act_err(ELU, e)
        out["b"] = (e, (err * (1 + rr) + rr * e.abs()) * (1 + U8) + U8 * e.abs())
    else:
        assert st.act == GELU
        g = act64(GELU, y)
        _, aa = act_err(GELU, y)
        out["b"] = (g, (GELU_SLOPE * err + aa) * (1 + U8) + U8 * g.abs())
    return out


def act_ref(st, x):
    """(ref, bound, exact) of bf16(act(x))."""
    if st.act in (NONE, RELU):
        return act64(st.act, x).to(F32).to(BF16).to(F64), None, True
    e = act64(st.act, x)
    r, _ = act_err(st.act, e)
    return e, r * e.abs() * (1 + U8) + U8 * e.abs(), False


def gate_refb(x_true, dtype, C, act=TANH):
    """act(f) sigmoid(g) of the gate input's true channels (dtype: the recorded input's, for the kernel's error)."""
    a, s, _ = gate_ref(x_true, C, act)
    return a * s, gate_fwd_err(x_true.to(dtype), C, act)


def decode_ref(st, q, k, v, p, strict):
    """o [n, H * dv] and its bound: q [n, H * dk], keys / values [n, p + 1, H * d] (row p: this step's)."""
    n = q.shape[0]
    H = st.H
    q4 = q.reshape(n, H, st.dk)
    k4 = k.reshape(n, -1, H, st.dk).permute(0, 2, 1, 3)
    v4 = v.reshape(n, -1, H, st.dv).permute(0, 2, 1, 3)
    o, b = decode_row(q4, k4, v4, p, strict, st.dk, st.qs)
    return o.reshape(n, -1), SAFETY * b.reshape(n, -1)


def ln_ref(st, x, eps=1e-5):
    r = ln_fwd_reference(x, st.g.detach().to(x.device), st.be.detach().to(x.device), eps)
    return r["y"], r["b_y"] * (1 + U8) + U8 * r["y"].abs()


def conv_small_ref(st, patch):
    """The window convolution's [n kh kw, Cout] output and bound (pg_conv_small_fwd, same-size with padding k // 2)."""
    n = patch.shape[0]
    dy = torch.zeros(n * st.kh * st.kw, st.w64.shape[0], dtype=F64)
    r = conv_reference(patch, st.w64, st.b64, dy, (st.kh // 2, st.kw // 2))
    return r["out"], r["b_out"]


# ----------------------------------------------------------------------------------------------------------------------
# chain: the stage references composed along the graph in float64
# ----------------------------------------------------------------------------------------------------------------------
def _eval64(env, st, p):
    """A stage's float64 value from the graph's float64 sources."""
    if st.kind == "virtual":
        return {"f": env.ev(st.src, p)}
    if st.kind == "conv_small":
        patch = env.ev(st.src, p)
        y = F.conv2d(patch, st.wx, st.b64, padding=(st.kh // 2, st.kw // 2))
        return {"f": y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])}
    a = env.ev(st.src, p)
    if st.kind == "linear":
        y = a @ st.wx.T + st.b64
        for r in st.res:
            y = y + env.ev(r, p)
        return {"f": y, "b": act64(st.act, y)}
    if st.kind == "act":
        return {"b": act64(st.act, a)}
    if st.kind == "gate":
        C = a.shape[1] // 2
        return {"b": torch.tanh(a[:, :C]) * torch.sigmoid(a[:, C:])}
    if st.kind == "gated_res":
        C = a.shape[1] // 2
        return {"f": env.ev(st.res[0], p) + a[:, :C] * torch.sigmoid(a[:, C:])}
    if st.kind == "ln":
        return {"b": F.layer_norm(a, (a.shape[1],), st.g.to(F64), st.be.to(F64), 1e-5)}
    if st.kind == "decode":
        q, k, v = _qkv(env, st, p, a)
        n = q.shape[0]
        if st.strict and p == 0:  # no visible key: the kernels define o = 0
            return {"b": torch.zeros(n, st.H * st.dv, dtype=F64)}
        kk = torch.stack([*[env.cache_row(st.kc, r) for r in range(p)], k], 1)
        vv = torch.stack([*[env.cache_row(st.vc, r) for r in range(p)], v], 1)
        q4 = q.reshape(n, st.H, 1, st.dk)
        k4 = kk.reshape(n, p + 1, st.H, st.dk).permute(0, 2, 1, 3)
        v4 = vv.reshape(n, p + 1, st.H, st.dv).permute(0, 2, 1, 3)
        s = (q4 @ k4.transpose(-1, -2)) / math.sqrt(st.dk)
        if st.strict:
            s[..., p] = -math.inf
        o = torch.softmax(s, -1) @ v4
        return {"b": o.reshape(n, -1)}
    raise AssertionError(st.kind)


def _qkv(env, st, p, q_src):
    """(q, k_new, v_new) true channels of a decode stage: q from its operand, k / v from its kv stage's value."""
    kv = env.value(p, st.kv, "b")
    if st.kv == st.src[1]:  # ImageGPT: one q | k | v projection
        C = st.H * st.dk
        return kv[:, :C], kv[:, C:2 * C], kv[:, 2 * C:]
    return q_src, kv[:, :st.dk], kv[:, st.dk:]


def chain(G, canvas):
    """The logits [n, cout] of every pixel of the final `canvas` (float64), the stage references composed along G."""
    env = Env(G, canvas.to(F64), exact=True)
    out = []
    for p in range(G.S):
        for st in G.stages:
            env.vals[p][st.name] = _eval64(env, st, p)
        out.append(env.vals[p]["logits"]["f"])
    return torch.stack(out, 2).reshape(canvas.shape[0], -1, G.h, G.w)
