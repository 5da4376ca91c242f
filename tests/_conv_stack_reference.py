"""The pixel-major stages of GatedPixelCNN, PixelSNAIL, VAE / BetaVAE, VQ-VAE and VQ-VAE-2 (models/gated_pixel_cnn.py,
models/pixel_snail.py, models/vae.py, models/vq_vae.py, models/vq_vae_2.py on nn/pm.py, nn/modules.py and nn/vq.py): a
stage table, float64 references of every stage, element-wise bounds and the hand-offs between stages.  Shared by
tests/test_conv_stack_bounds_cpu.py and tests/test_conv_stack_stages_gpu.py; not a test module.

GatedPixelCNN's table is a stage graph read from the state dict along oracle/reference_path.py `_gated_layer`: every
stage names its sources (`src`, summed when there are several), its residual (the output of the stage `res` names, in
that stage's dtype), its taps (padding plus the front crop), its input activation and its emit mode.  Besides the
convolutions it holds the two gates of each layer, the input layer's direct image convolutions (kind `image`) and its
cast.  `forward_handoffs` and `backward_handoffs` hold the recorded tensors passed between stages to that graph, and
`graph_chain` composes the stage references along it in float64.  PixelSNAIL's graph follows `pixel_snail_forward`
and `_snail_residual` the same way, with three more kinds: `gated_res` (the identity gate plus the fp32 residual),
`attention` (the causal attention block on [position | features | image | 0-pad], checked sub-step by sub-step) and
`stream` (the fp32 sum s + out, which no Function records; it is held at its hand-offs).

Stage table.  `table(state)` reads the layer structure from a state dict with the helpers of the reference restatements
(tests/_vae_reference.py, tests/_vq_vae_reference.py), never from the arguments the product passes, so a wrong
argument fails.  One entry per convolution, keyed by its parameter prefix: its kind (conv, strided, transposed), stride
and padding, the reference's activation in front of it (`in_act`), whether its output leaves through an activation it
owns (`act`: the strided convolutions' ReLU, a non-last transposed convolution's ReLU), and the stage whose input is its
residual (`res`: the input of a residual block).  Where the reference applies ReLU to a ReLU output (the first residual
block after a strided convolution) ReLU is the identity on the stage's input and `in_act` is none.

References.  Each stage is computed in float64 from the product's recorded inputs: the activation it read (rounded by
the table's `in_act` to the bf16 operand DESIGN §3 names), the residual the table names, the weight rounded to bf16
and the fp32 bias; backward from the recorded incoming gradient, taken through the stage's own activation from its
recorded activated output and rounded to the bf16 GEMM operand.  It gives the main output, the activated output,
dx (through the input activation's derivative, taken from the bf16 operand), dw, db and dres.

Bounds (U24 = 2^-24, U8 = 2^-8 the unit roundoffs of fp32 and bf16).  A contraction of K products summed in fp32 is
within (K + 2) U24 of its magnitude (tests/_gemm_reference.py); a split-K weight gradient adds at most 64 + 132 + 1
roundings (one k-block of padding, one per slice, one for the output); a scatter of T taps adds T; a dgrad whose
per-tap partials are stored in bf16 before the scatter (pg_tap_gather and pg_strided_gather paths) adds U8 of the
magnitude.  An output stored in bf16 adds U8 of itself; ReLU and ELU are 1-Lipschitz, so an activated output
inherits its input's bound (ELU adds its kernel error, tests/_act_reference.act_err).  A gradient the reference passes
through unchanged is bit-exact: dres (in the residual's dtype) and every pad column of every output and gradient,
which must be +0.0."""

import collections

import torch
from torch.nn import functional as F

import _vae_reference as V
import _vq_vae_reference as VQ
from _act_reference import ELU as ACT_ELU, NONE as ACT_NONE, TANH as ACT_TANH, act_err, gate_bwd, gate_fwd_err, gate_ref
from _attention_reference import SAFETY, attention
from _gemm_reference import bound as gemm_bound
from oracle.reference_path import _count, causal_attention, causal_mask, gated_activation, image_positional_encoding

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U24, U8 = 2.0 ** -24, 2.0 ** -8
RELU, ELU, NONE = "relu", "elu", None

IDENT = "identity"  # an emitted plain bf16 copy
# kind: conv, strided, transposed (a Function of nn/pm.py), image (`pm.image_conv` of the NCHW image: the direct fp32
# kernel or `conv`), gate, act_cast;  act: the mode of the activated output `ya` (post, companion, pre_grad; None: no
# `ya`) and emit its activation;  res: the stage feeding the residual, its input (res_of "in") or its output ("out");
# f32: the main output is fp32 (True), bf16 (False) or not written (None);  src: the stages whose outputs, summed, are
# this stage's input ("image": the model input);  mask: the weight is multiplied by the reference's causal_mask (a
# mask-centre CausalConv2d);  attn: an attention stage's Attn.
# PixelSNAIL adds the kinds gated_res (an identity gate plus a fp32 residual), attention (the causal attention block on
# [position | features | image | 0-pad]) and stream (the fp32 sum of a block's input and its output).
Layer = collections.namedtuple("Layer", "kind stride pad in_act act res emit f32 src res_of mask attn",
                               defaults=(1, 0, NONE, None, None, None, None, (), "in", False, None))
# C feature channels, c_img image channels, key / value channels of the one head, strict (mask-centre) attention
Attn = collections.namedtuple("Attn", "C c_img key value strict")


# ----------------------------------------------------------------------------------------------------------------------
# stage table
# ----------------------------------------------------------------------------------------------------------------------
def _res_stack(T, key, n_blocks, post_act):
    for b in range(n_blocks):
        k = f"{key}._net.{b}._net"
        T[f"{k}.1"] = Layer("conv", 1, 1, NONE if (post_act and b == 0) else RELU, "companion", None, RELU)
        T[f"{k}.3"] = Layer("conv", 1, 0, RELU, None, f"{k}.1")


def _encoder(T, state, key):
    k = V._n_strided(state, key + ".")
    for j in range(k):
        T[f"{key}.{2 * j}"] = Layer("strided", 2, 1, NONE, "post", None, RELU)
    _res_stack(T, f"{key}.{2 * k}", VQ._n_blocks(state, f"{key}.{2 * k}"), k > 0)
    T[f"{key}.{2 * k + 1}"] = Layer("conv", 1, 1, RELU, None, None)


def _decoder(T, state, key):
    T[f"{key}.0"] = Layer("conv", 1, 1, NONE, None, None)
    _res_stack(T, f"{key}.1", VQ._n_blocks(state, f"{key}.1"), False)
    k = V._n_strided(state, key + ".")
    j = 2
    for t in range(k):
        T[f"{key}.{j}"] = Layer("transposed", 2, 1, RELU if t == 0 else NONE, "post" if t < k - 1 else None, None,
                                 RELU if t < k - 1 else None)
        j += 2 if t < k - 1 else 1


def _gated_layer(T, state, pre, prv):
    """One GatedPixelCNN layer (oracle/reference_path.py `_gated_layer`); prv: the previous layer, None for the causal
    input layer, which reads the image.  Kernel size and padding come from the weight shapes as the restatement's."""
    k = state[pre + "._vstack_1xN.weight"].shape[-1]
    p = (k - 1) // 2
    causal = prv is None
    conv = lambda src, pad, res=None, f32=False, **kw: Layer("conv", 1, pad, src=src, res=res, res_of="out", f32=f32,
                                                             **kw)
    image = lambda pad: Layer("image", 1, pad, f32=True, src=("image",))
    if causal:
        T[pre + "._vstack_1xN"] = image((0, p))
        T[pre + ":act_cast"] = Layer("act_cast", src=(pre + "._vstack_1xN",))
        T[pre + "._vstack_Nx1"] = conv((pre + ":act_cast",), (p + 1, 0))
    else:
        T[pre + "._vstack_1xN"] = conv((prv + ":gate_v",), (0, p))
        T[pre + "._vstack_Nx1"] = conv((pre + "._vstack_1xN",), (p + 1, 0))
    T[pre + "._link"] = conv((pre + "._vstack_Nx1",), (0, 0))
    if causal:  # the image convolutions' sums with v2 and the link are the gates' inputs: fp32
        T[pre + "._vstack_1x1"] = image((0, 0))
        T[pre + "._hstack_1xN"] = image((0, p + 1))
        T[pre + ":gate_v"] = Layer("gate", src=(pre + "._vstack_Nx1", pre + "._vstack_1x1"))
        T[pre + ":gate_h"] = Layer("gate", src=(pre + "._link", pre + "._hstack_1xN"))
    else:  # a later layer adds them in the GEMM epilogues: bf16 residuals
        T[pre + "._vstack_1x1"] = conv((prv + ":gate_v",), (0, 0), pre + "._vstack_Nx1")
        T[pre + "._hstack_1xN"] = conv((prv + "._hstack_residual",), (0, p), pre + "._link")
        T[pre + ":gate_v"] = Layer("gate", src=(pre + "._vstack_1x1",))
        T[pre + ":gate_h"] = Layer("gate", src=(pre + "._hstack_1xN",))
    T[pre + "._hstack_skip"] = conv((pre + ":gate_h",), (0, 0), None if causal else prv + "._hstack_skip", f32=True)
    T[pre + "._hstack_residual"] = conv((pre + ":gate_h",), (0, 0), None if causal else prv + "._hstack_residual",
                                        f32=True, act="companion", emit=IDENT)


def _gated_pixel_cnn(state):
    """The stage graph of oracle/reference_path.py `gated_pixel_cnn_forward`: the causal input layer, the gated layers
    and the head (ReLU, 1x1, ReLU, 1x1; the first 1x1 emits its ReLU for the second, pre_grad)."""
    T = {}
    _gated_layer(T, state, "_input", None)
    prv = "_input"
    for i in range(_count(state, "_gated_layers")):
        _gated_layer(T, state, f"_gated_layers.{i}", prv)
        prv = f"_gated_layers.{i}"
    T["_head.1"] = Layer("conv", 1, (0, 0), RELU, "pre_grad", None, RELU, None, (prv + "._hstack_skip",), "out")
    T["_head.3"] = Layer("conv", 1, (0, 0), RELU, None, None, None, True, ("_head.1",), "out")
    return T


def _pixel_snail(state):
    """The stage graph of oracle/reference_path.py `pixel_snail_forward` and `_snail_residual`: the mask-centre 3x3
    input convolution; per residual block conv2x2(elu) emitting elu for conv2x2(elu), whose 2C outputs an identity gate
    adds to the block input; per block the features' cast, the attention on [position | features | image | 0-pad],
    the ELU-in / ELU-out 1x1 convolutions `_residual_out`, `_attention_out` and `_out` (reading the sum of the first
    two) and the fp32 stream s + out; the head's two 1x1 convolutions, the second one to fp32 logits."""
    T = {}
    C, c_img = state["_input.weight"].shape[:2]
    T["_input"] = Layer("image", 1, (1, 1), f32=True, src=("image",), mask=True)
    s = "_input"
    for i in range(_count(state, "_pixel_snail_blocks")):
        blk = f"_pixel_snail_blocks.{i}"
        res = s
        for j in range(_count(state, blk + "._residual")):
            pre = f"{blk}._residual.{j}"
            T[pre + "._input_conv"] = Layer("conv", 1, (1, 1), ELU, "pre_grad", None, ELU, None, (res,), "out")
            T[pre + "._output_conv"] = Layer("conv", 1, (1, 1), ELU, None, None, None, False, (pre + "._input_conv",),
                                             "out")
            T[pre + ":gated_res"] = Layer("gated_res", f32=True, src=(pre + "._output_conv",), res=res, res_of="out")
            res = pre + ":gated_res"
        att = blk + "._attention"
        T[blk + ":act_cast"] = Layer("act_cast", src=(res,))
        T[att] = Layer("attention", f32=True, src=(blk + ":act_cast",),
                       attn=Attn(C, c_img, state[att + "._q.weight"].shape[0], state[att + "._proj.weight"].shape[0],
                                 True))
        post = lambda *src: Layer("conv", 1, (0, 0), ELU, "post", None, ELU, None, src, "out")
        T[blk + "._residual_out"] = post(res)
        T[blk + "._attention_out"] = post(att)
        T[blk + "._out"] = post(blk + "._residual_out", blk + "._attention_out")
        T[blk + ":stream"] = Layer("stream", f32=True, src=(s, blk + "._out"))
        s = blk + ":stream"
    T["_output.0"] = Layer("conv", 1, (0, 0), NONE, None, None, None, False, (s,), "out")
    T["_output.1"] = Layer("conv", 1, (0, 0), NONE, None, None, None, True, ("_output.0",), "out")
    return T


def table(state):
    """{stage name: Layer} of a VAE, VQ-VAE, VQ-VAE-2, GatedPixelCNN or PixelSNAIL state dict, in the reference's
    forward order.  A convolution is named by its parameter prefix; a stage without parameters by its layer and its
    role."""
    T = {}
    tops = sorted({k.split(".")[0] for k in state})
    if "_gated_layers" in tops or "_input" in tops and "_input._vstack_1xN.weight" in state:
        return _gated_pixel_cnn(state)
    if "_input.weight" in state and "_output.1.weight" in state:
        return _pixel_snail(state)
    if "_encoder" in tops and any(k.startswith("_encoder.0.") for k in state):  # VAE: Sequentials of stages
        for i in range(V._count(state, "_encoder.")):
            _encoder(T, state, f"_encoder.{i}._net")
        for i in range(V._count(state, "_decoder.")):
            _decoder(T, state, f"_decoder.{i}._net")
        return T
    if "_encoder" in tops:  # VQ-VAE
        _encoder(T, state, "_encoder._net")
        T["_quantizer._net.0"] = Layer("conv", 1, 0, NONE, None, None)
        _decoder(T, state, "_decoder._net")
        return T
    _encoder(T, state, "_encoder_b._net")
    _encoder(T, state, "_encoder_t._net")
    T["_quantizer_t._net.0"] = Layer("conv", 1, 0, NONE, None, None)
    _decoder(T, state, "_decoder_t._net")
    T["_conv"] = Layer("conv", 1, 0, NONE, None, None)
    T["_quantizer_b._net.0"] = Layer("conv", 1, 0, NONE, None, None)
    _decoder(T, state, "_decoder_b._net")
    return T


# ----------------------------------------------------------------------------------------------------------------------
# checks
# ----------------------------------------------------------------------------------------------------------------------
class Checks:
    """Collects |got - ref| / bound per named check, and the failures."""

    def __init__(self):
        self.ratios, self.failures = {}, {}

    def within(self, name, got, ref, bound):
        got = got.detach().to(F64).cpu()
        ref, bound = ref.detach().to(F64).cpu(), bound.detach().to(F64).cpu()
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        err = (got - ref).abs()
        bad = ~(err <= bound)  # NaN fails
        exact = bound == 0
        # an exact element (zero bound) counts 0 when it matches, infinity when it does not
        ratio = torch.where(exact, torch.where(err > 0, float("inf"), 0.0), err / bound.clamp_min(1e-300))
        self.ratios[name] = float(ratio.max()) if ratio.numel() else 0.0
        if bool(bad.any()):
            i = int(bad.flatten().nonzero()[0])
            self.failures[name] = (f"{name}: {int(bad.sum())} of {bad.numel()} outside the bound; first at {i}: got "
                                   f"{got.flatten()[i]:.6e}, ref {ref.flatten()[i]:.6e}, bound {bound.flatten()[i]:.3e}")

    def equal(self, name, got, ref):
        """Bit for bit, dtype included."""
        ok = got.dtype == ref.dtype and got.shape == ref.shape and torch.equal(_bits(got), _bits(ref.to(got.device)))
        self.ratios[name] = 0.0 if ok else float("inf")
        if not ok:
            self.failures[name] = f"{name}: not bit-identical ({got.dtype} {tuple(got.shape)} vs {ref.dtype} {tuple(ref.shape)})"

    def zero(self, name, t):
        """Every element +0.0 (the bits of zero)."""
        if t is None or t.numel() == 0:
            return
        ok = not bool(_bits(t).any())
        self.ratios[name] = 0.0 if ok else float("inf")
        if not ok:
            self.failures[name] = f"{name}: {int((_bits(t) != 0).sum())} pad elements are not +0.0"

    def failed_kinds(self):
        return {kind_of(n) for n in self.failures}

    def worst_by_kind(self):
        out = {}
        for n, r in self.ratios.items():
            out[kind_of(n)] = max(out.get(kind_of(n), 0.0), r)
        return out


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def kind_of(name):
    """'<stage kind>.<output>' of a check name '<stage kind> <parameter prefix>.<output>'."""
    kind, rest = name.split(" ", 1)
    return f"{kind}.{rest.rsplit('.', 1)[1]}"


# ----------------------------------------------------------------------------------------------------------------------
# convolution stages
# ----------------------------------------------------------------------------------------------------------------------
def nchw(t, geom, c):
    n, h, w = geom
    return t[:, :c].to(F64).reshape(n, h, w, c).permute(0, 3, 1, 2)


def pm(t):
    n, c, h, w = t.shape
    return t.permute(0, 2, 3, 1).reshape(n * h * w, c)


def _dact_out(act, a):
    """act'(pre) from the activated value a = act(pre): ReLU's 1[a > 0], ELU's 1 or a + 1."""
    a = a.to(F64)
    if act == ELU:
        return torch.where(a > 0, torch.ones_like(a), a + 1)
    assert act == RELU, act
    return (a > 0).to(F64)


def act64(act, y):
    """ReLU, ELU, or the identity (no activation, or an emitted plain copy)."""
    assert act in (RELU, ELU, NONE, IDENT), act
    if act == ELU:
        return F.elu(y)
    return torch.relu(y) if act == RELU else y


def _elu_store(ref, err):
    """Bound of bf16(kernel elu(y~)) for |y~ - y| <= err and ref = elu(y): ELU is 1-Lipschitz, the kernels' fp32 ELU is
    within act_err(ELU) of its value (tests/_act_reference.py), then one bf16 rounding."""
    r, _ = act_err(ACT_ELU, ref)
    return _bf16_store(ref, err * (1 + r) + r * ref.abs())


def _linear(layer, x, w):
    if layer.kind == "transposed":
        return F.conv_transpose2d(x, w, None, stride=layer.stride, padding=layer.pad)
    y = F.conv2d(x, w, None, stride=layer.stride, padding=layer.pad)
    # a stride-1 convolution keeps its input's size: the front crop of the padded output (the reference's [:h, :w])
    return y[:, :, : x.shape[2], : x.shape[3]] if layer.stride == 1 else y


def stage_in(layer, x):
    """What the stage's contraction reads: its input activation applied to x."""
    return act64(layer.in_act, x)


def stage_y(layer, xa, w, b, res=None):
    """The stage's output before any activation: the contraction of xa, the bias and the residual."""
    y = _linear(layer, xa, w) + b[None, :, None, None]
    return y if res is None else y + res


def stage_out(layer, y):
    """What the next stage receives: emit(y) when the stage's activated output is a true post-activation output, else y
    (a companion is a copy; a pre_grad output stands for y and its activation is the consumer's in_act)."""
    return act64(layer.emit, y) if layer.act == "post" else y


def _bf16_store(ref, err):
    """Bound of a bf16 store of a value within err of ref."""
    return err * (1 + U8) + U8 * ref.abs()


def conv_stage(C, name, layer, rec, res_in, weight, bias, res_dtype=None, operand_given=False):
    """Holds one recorded convolution to its float64 reference.  rec: the Recorder's record (args, out, grads, res);
    res_in: the table's residual (or None) and res_dtype the dtype the table gives it (None: the recorded one);
    operand_given: the input is a pre_grad output, already activated, so the operand is the input itself."""
    label = f"{layer.kind} {name}"
    x, xa_got = rec.x, rec.xa
    in_geom, out_geom = rec.in_geom, rec.out_geom
    w64 = weight.detach().to(BF16).to(F64)
    b64 = bias.detach().to(F64)
    if layer.kind == "transposed":
        cin, cout = w64.shape[:2]
    else:
        cout, cin = w64.shape[:2]
    kh, kw = w64.shape[-2:]
    T = kh * kw

    # the operand: bf16(in_act(x)) bit for bit (ELU: within its kernel error and one rounding), or x itself
    if operand_given:
        C.equal(f"{label}.xa", xa_got[:, :cin], x[:, :cin])
    elif layer.in_act == ELU:
        e = act64(ELU, x[:, :cin].to(F64))
        C.within(f"{label}.xa", xa_got[:, :cin], e, _elu_store(e, torch.zeros_like(e)))
    else:
        C.equal(f"{label}.xa", xa_got[:, :cin], (torch.relu(x.float()) if layer.in_act == RELU else x.float())
                [:, :cin].to(BF16))
    C.zero(f"{label}.xa_pad", xa_got[:, cin:])
    xa64 = nchw(xa_got, in_geom, cin).clone().requires_grad_(True)
    wv = w64.clone().requires_grad_(True)
    r64 = None if res_in is None else nchw(res_in, out_geom, cout)
    y64 = stage_y(layer, xa64, wv, b64, r64)
    mag = stage_y(layer, xa64.detach().abs(), w64.abs(), b64.abs(), None if r64 is None else r64.abs())
    k_fwd = cin * (T if layer.kind != "transposed" else 1) + (T if layer.kind == "transposed" else 0)
    y, err = pm(y64.detach()), pm((k_fwd + 3) * U24 * mag)

    main, ya = rec.y, rec.ya
    if main is not None:
        if layer.f32 is not None and main.dtype != (F32 if layer.f32 else BF16):
            C.failures[f"{label}.y"] = f"{label}.y: stored in {main.dtype}, the table gives {'fp32' if layer.f32 else 'bf16'}"
        if main.dtype == F32:
            C.within(f"{label}.y", main[:, :cout], y, err)
        else:
            C.within(f"{label}.y", main[:, :cout], y, _bf16_store(y, err))
        C.zero(f"{label}.y_pad", main[:, cout:])
    if ya is not None:
        act = act64(layer.emit, y)  # ReLU is 1-Lipschitz: the activated output inherits y's bound
        C.within(f"{label}.ya", ya[:, :cout], act, _elu_store(act, err) if layer.emit == ELU else _bf16_store(act, err))
        C.zero(f"{label}.ya_pad", ya[:, cout:])

    # backward: the gradient w.r.t. y, as the bf16 GEMM operand
    if rec.grads is None:
        return
    g = None
    for gi, wrt in zip(rec.grads, (main, ya)):
        if gi is None:
            continue
        if wrt is ya and layer.act == "post" and layer.emit == ELU:
            gi = _post_elu_operand(C, label, gi[:, :cout], ya[:, :cout], rec.dact)
        else:
            gi = gi[:, :cout].to(F64)
            if wrt is ya and layer.act == "post":  # the stage's own activation, from its activated output
                gi = gi * _dact_out(layer.emit, ya[:, :cout])
        g = gi if g is None else g + gi
    if g is None:
        return
    gb = g.to(F32).to(BF16).to(F64)
    gb4 = nchw(gb, out_geom, cout)
    dxa, dw = torch.autograd.grad(y64, (xa64, wv), gb4, retain_graph=True)
    xa_abs = xa64.detach().abs().requires_grad_(True)
    w_abs = w64.abs().requires_grad_(True)
    mag_x, mag_w = torch.autograd.grad(_linear(layer, xa_abs, w_abs), (xa_abs, w_abs), gb4.abs())
    P_out, P_in = gb.shape[0], xa_got.shape[0]
    dx_g, dw_g, db_g, dres_g = rec.dx, rec.dw, rec.db, rec.dres

    if dw_g is not None:
        k_w = (P_out if layer.kind != "transposed" else P_in) + 64 + 132 + 3
        C.within(f"{label}.dw", dw_g, dw, k_w * U24 * mag_w)
    if db_g is not None:
        C.within(f"{label}.db", db_g, gb.sum(0), (P_out + 64 + 132 + 3) * U24 * gb.abs().sum(0))
    if dx_g is not None:
        d = pm(dxa)
        m = pm(mag_x)
        k_x = cout * T + T + 3
        if layer.in_act in (RELU, ELU):  # the input activation's derivative, from the bf16 operand
            f = _dact_out(layer.in_act, xa_got[:, :cin])
            d, m = d * f, m * f
            k_x += 2 if layer.in_act == ELU else 0  # the fp32 xa + 1 and its product
        err = k_x * U24 * m
        if rec.bf16_partials:
            err = err + U8 * m
        if dx_g.dtype == BF16:
            err = _bf16_store(d, err)
        C.within(f"{label}.dx", dx_g[:, :cin], d, err)
        C.zero(f"{label}.dx_pad", dx_g[:, cin:])
    if rec.has_res:
        # d res = dy: the incoming gradient itself, in the residual's dtype
        C.equal(f"{label}.dres", dres_g if dres_g is not None else torch.empty(0), g.to(res_dtype or rec.res_dtype))


def _post_elu_operand(C, label, dya, ya, got):
    """The bf16 operand bf16(dya (ya + 1)) (1 where ya > 0) that _lib.dact_from_out forms in fp32 from the gradient of
    an ELU POST output: the recorded one (`got`, [P, >= cout] bf16) against float64, within U24 |dya| for the rounding
    of ya + 1, 2 U24 of itself for the product and one bf16 rounding; returned in float64 as the operand the
    contraction checks read.  Without a record (the backward skipped ELU'), the float64 operand rounded to bf16."""
    d64 = dya.to(F64)
    ref = d64 * _dact_out(ELU, ya)
    if got is None:
        C.failures[f"{label}.dya"] = f"{label}.dya: the POST output's gradient never went through dact_from_out"
        C.ratios[f"{label}.dya"] = float("inf")
        return ref.to(F32).to(BF16).to(F64)
    cout = ref.shape[1]
    C.within(f"{label}.dya", got[:, :cout], ref, _bf16_store(ref, U24 * d64.abs() + 2 * U24 * ref.abs()))
    C.zero(f"{label}.dya_pad", got[:, cout:])  # the padded dy operand's columns
    return got[:, :cout].to(F64)


# ----------------------------------------------------------------------------------------------------------------------
# latent, quantizer and MSE stages
# ----------------------------------------------------------------------------------------------------------------------
def latent_stage(C, rec):
    h, eps, L = rec.args[1], rec.args[2], rec.args[3]
    n = eps.shape[0]
    e = pm(eps.to(F64))
    m, s = h[:, :L].to(F64), h[:, L: 2 * L].to(F64)
    es = torch.exp(s)
    z = m + es * e
    z_err = 8 * U24 * (m.abs() + (es * e).abs())
    z_got, kl_got = rec.out
    C.within("latent _latent.z", z_got[:, :L], z, _bf16_store(z, z_err))
    C.zero("latent _latent.z_pad", z_got[:, L:])
    t = -0.5 * (1 + 2 * s - es ** 2 - m ** 2)
    ta = 0.5 * (1 + 2 * s.abs() + es ** 2 + m ** 2)
    per = h.shape[0] // n
    C.within("latent _latent.kl", kl_got, t.reshape(n, -1).sum(1), (per * L + 8) * U24 * ta.reshape(n, -1).sum(1))
    if rec.grads is None:
        return
    dz, dkl = rec.grads
    d = torch.zeros_like(m) if dz is None else dz[:, :L].to(BF16).to(F64)
    g = torch.zeros(h.shape[0], 1, dtype=F64) if dkl is None else dkl.to(F64).repeat_interleave(per)[:, None]
    g = g.to(d.device)
    dm = d + g * m
    ds = d * es * e + g * (es ** 2 - 1)
    dh = rec.res[0]
    C.within("latent _latent.dx_mean", dh[:, :L], dm, _bf16_store(dm, 4 * U24 * (d.abs() + (g * m).abs())))
    C.within("latent _latent.dx_logstd", dh[:, L: 2 * L], ds,
             _bf16_store(ds, 8 * U24 * ((d * es * e).abs() + (g * (es ** 2 + 1)).abs())))


def assign_bound(xd, ed):
    """|fl(dist) - dist| <= (d + 3) u (|x|^2 + |e|^2 + 2 sum |x_j e_j|) per code: the fp32 rounding of the quantizer's
    distances (pg_vq_assign), [P, K] in float64."""
    d = xd.shape[1]
    return (d + 3) * U24 * ((xd * xd).sum(1, keepdim=True) + (ed * ed).sum(1) + 2 * xd.abs() @ ed.abs().t())


def quantizer_stage(C, name, rec):
    """The straight-through operand, the commitment loss and dz of one recorded quantizer call."""
    label = f"quantizer {name}"
    z_grad, z, emb_param, left, vq, width, out_dtype = rec.args
    emb = rec.emb  # the codebook the loss used (before any EMA update)
    d = emb.shape[1]
    out, loss = rec.out
    xd, ed = z[:, :d].to(F64), emb.to(F64)
    idx = rec.idx.long()
    dist = (xd * xd).sum(1, keepdim=True) + (ed * ed).sum(1) - 2 * xd @ ed.t()
    bound = assign_bound(xd, ed)
    C.within(f"{label}.idx", dist.gather(1, idx[:, None])[:, 0], dist.min(1).values,
             bound.gather(1, idx[:, None])[:, 0] + bound.max(1).values)
    c0 = 0 if left is None else left.shape[1]
    q = ed[idx]
    st = (z[:, :d] + (emb[idx] - z[:, :d])).to(out_dtype)
    C.equal(f"{label}.out", out[:, c0: c0 + d], st)
    if left is not None:
        C.equal(f"{label}.left", out[:, :c0], left)
    C.zero(f"{label}.out_pad", out[:, c0 + d:])
    numel = z.shape[0] * d
    two = 1 if vq._use_ema else 2
    ref = two * ((xd - q) ** 2).sum() / numel
    C.within(f"{label}.loss", loss.reshape(1), ref.reshape(1), (numel + 4) * U24 * ref.abs().reshape(1))
    if rec.grads is None:
        return
    dout, dloss = rec.grads
    dq = torch.zeros_like(xd) if dout is None else dout[:, c0: c0 + d].to(z_grad.dtype).to(F64)
    g = 0.0 if dloss is None else float(dloss)
    c = (xd - q) * (2.0 / numel) * g
    dz_ref = dq + c
    err = 4 * U24 * (dq.abs() + c.abs())
    dz = rec.res[0]
    if dz.dtype == BF16:
        err = _bf16_store(dz_ref, err)
    C.within(f"{label}.dx", dz[:, :d], dz_ref, err)
    C.zero(f"{label}.dx_pad", dz[:, d:])


def mse_stage(C, rec):
    a, b, cols, numel = rec.args
    diff = a[:, :cols].to(F64) - b[:, :cols].to(F64)
    ref = (diff ** 2).sum() / numel
    C.within("mse _mse.loss", rec.out.reshape(1), ref.reshape(1), (numel + 4) * U24 * ref.reshape(1))
    if rec.grads is None:
        return
    (g,) = rec.grads
    da_ref = diff * (2.0 / numel) * float(g)
    da, db = rec.res[0], rec.res[1]
    C.within("mse _mse.dx", da[:, :cols], da_ref, 4 * U24 * da_ref.abs())
    C.equal("mse _mse.db", db, -da)
    C.zero("mse _mse.dx_pad", da[:, cols:])


# ----------------------------------------------------------------------------------------------------------------------
# the stage chain: the references above composed along the table, in float64 on their own outputs
# ----------------------------------------------------------------------------------------------------------------------
def _segment(T, P, prefix, x):
    """The table's stages under `prefix`, in order: each reads the previous one's stage_out, and a stage with a `res`
    adds the input of the stage it names."""
    inputs = {}
    for name, layer in T.items():
        if name != prefix and not name.startswith(prefix + "."):
            continue
        inputs[name] = x
        res = inputs[layer.res] if layer.res else None
        x = stage_out(layer, stage_y(layer, stage_in(layer, x), P[name + ".weight"], P[name + ".bias"], res))
    return x


def _quantize(z, emb, use_ema=True):
    """The quantizer stage: the nearest code (float64 distances), the straight-through value and the loss."""
    n, d, h, w = z.shape
    flat = z.permute(0, 2, 3, 1).reshape(-1, d)
    e = emb.detach() if use_ema else emb
    idx = ((flat * flat).sum(1, keepdim=True) + (e * e).sum(1) - 2 * flat @ e.t()).argmin(1)
    q = e[idx].reshape(n, h, w, d).permute(0, 3, 1, 2)
    loss = ((z - q.detach()) ** 2).mean()
    if not use_ema:
        loss = loss + ((q - z.detach()) ** 2).mean()
    return z + (q - z).detach(), loss


def chain(cls, T, P, x, eps=None):
    """The model's two outputs, composed from the stage references along the table T: (logits, kl) of a VAE,
    (x_hat, vq_loss) of VectorQuantizedVAE / VectorQuantizedVAE2.  P: parameters and buffers by name."""
    if cls == "VAE":
        h = x
        for i in range(V._count(P, "_encoder.")):
            h = _segment(T, P, f"_encoder.{i}._net", h)
        L = eps.shape[1]
        mean, log_std = h[:, :L], h[:, L: 2 * L]
        kl = (-0.5 * (1 + 2 * log_std - torch.exp(log_std) ** 2 - mean ** 2)).sum((1, 2, 3))
        z = mean + torch.exp(log_std) * eps
        for i in range(V._count(P, "_decoder.")):
            z = _segment(T, P, f"_decoder.{i}._net", z)
        return z, kl
    if cls == "VectorQuantizedVAE":
        z = _segment(T, P, "_quantizer._net.0", _segment(T, P, "_encoder._net", x))
        q, loss = _quantize(z, P["_quantizer._net.1._embedding"])
        return _segment(T, P, "_decoder._net", q), loss
    assert cls == "VectorQuantizedVAE2", cls
    eb = _segment(T, P, "_encoder_b._net", x)
    et = _segment(T, P, "_encoder_t._net", eb)
    qt, loss_t = _quantize(_segment(T, P, "_quantizer_t._net.0", et), P["_quantizer_t._net.1._embedding"])
    qb, loss_b = _quantize(_segment(T, P, "_quantizer_b._net.0", eb), P["_quantizer_b._net.1._embedding"])
    dt = _segment(T, P, "_decoder_t._net", qt)
    left = _segment(T, P, "_conv", dt)
    x_hat = _segment(T, P, "_decoder_b._net", torch.cat((left, qb), 1))
    return x_hat, 0.5 * (loss_b + loss_t) + ((dt - eb) ** 2).mean()


# ----------------------------------------------------------------------------------------------------------------------
# gate, image-convolution and act_cast stages
# ----------------------------------------------------------------------------------------------------------------------
def gate_stage(C, name, rec):
    """pm.gated with tanh: y = tanh(f) sigmoid(g) of the recorded x = [f | g] (fp32 on the input layer, bf16 after), and
    dx from the recorded incoming gradient in x's dtype (what the product hands pg_gated_act_bwd)."""
    label = f"gate {name}"
    x = rec.args[0]
    c = x.shape[1] // 2
    a, s, _ = gate_ref(x.to(F64), c, ACT_TANH)
    y, err = a * s, gate_fwd_err(x, c, ACT_TANH)
    C.within(f"{label}.y", rec.out, y, _bf16_store(y, err) if rec.out.dtype == BF16 else err)
    if rec.grads is None or rec.grads[0] is None:
        return
    ref_f, tol_f, ref_g, tol_g = gate_bwd(x, rec.grads[0].to(x.dtype), c, ACT_TANH, x.dtype)
    dx = rec.res[0]
    C.within(f"{label}.dx", dx, torch.cat((ref_f, ref_g), 1), torch.cat((tol_f, tol_g), 1))


def small_stage(C, name, layer, rec, weight, bias):
    """The direct fp32 convolution of the image (pm._SmallConv): y, dw and db against float64 from the recorded image and
    the table's padding, weight (fp32) and bias, never the ones the product passed.  Every product and sum is an fp32 fma: y sums K =
    Cin kh kw products after the bias, (K + 2) U24 of its magnitude; dw sums every pixel's product on one thread's chain
    and adds at most 2 x 132 block slices, (P + 268) U24; db is a column sum of P terms, (P + 4) U24.  dx is never
    asked for (the image needs no gradient).  dw is dense over masked taps, as the reference's."""
    label = f"small {name}"
    x = rec.args[0]
    n, cin, h, w = x.shape
    cout = weight.shape[0]
    x64 = x.detach().to(F64)
    wv = weight.detach().to(F64).clone().requires_grad_(True)
    lay = layer
    y64 = stage_y(lay, x64, wv, bias.detach().to(F64))
    mag = stage_y(lay, x64.abs(), wv.detach().abs(), bias.detach().to(F64).abs())
    K = cin * weight.shape[2] * weight.shape[3]
    C.within(f"{label}.y", rec.out, pm(y64.detach()), pm((K + 2) * U24 * mag))
    if rec.grads is None or rec.grads[0] is None:
        return
    g = rec.grads[0].to(F64)
    g4 = nchw(g, (n, h, w), cout)
    (dw,) = torch.autograd.grad(y64, (wv,), g4)
    wa = wv.detach().abs().requires_grad_(True)
    (mag_w,) = torch.autograd.grad(_linear(lay, x64.abs(), wa), (wa,), g4.abs())
    P = g.shape[0]
    C.within(f"{label}.dw", rec.res[1], dw, (P + 2 * 132 + 4) * U24 * mag_w)
    C.within(f"{label}.db", rec.res[2], g.sum(0), (P + 4) * U24 * g.abs().sum(0))


ACT_IDS = {0: NONE, 1: RELU}  # _lib activation ids of the act_cast records


def act_cast_stage(C, name, rec):
    """pm.act_cast: bf16(act(x)) bit for bit; its backward (an
    unactivated cast) hands the incoming gradient back in x's dtype, bit for bit."""
    label = f"act_cast {name}"
    x, act = rec.args[0], ACT_IDS[rec.args[1]]
    C.equal(f"{label}.y", rec.out, (torch.relu(x.float()) if act == RELU else x.float()).to(BF16))
    if rec.grads is not None and rec.grads[0] is not None and act is NONE:
        C.equal(f"{label}.dx", rec.res[0], rec.grads[0].to(x.dtype))


def gated_res_stage(C, name, rec, res_in):
    """pm.gated_res with the identity gate: y = res + f sigmoid(g) of the recorded bf16 x = [f | g] and the table's fp32
    residual, within gate_fwd_err and the fp32 add; dx from gate_bwd with bf16 x and the fp32 incoming gradient; dres
    is that gradient itself, bit for bit."""
    label = f"gated_res {name}"
    x = rec.args[0]
    c = x.shape[1] // 2
    a, s, _ = gate_ref(x.to(F64), c, ACT_NONE)
    y, err = res_in[:, :c].to(F64) + a * s, gate_fwd_err(x, c, ACT_NONE)
    C.within(f"{label}.y", rec.out, y, err + U24 * (y.abs() + err))
    if rec.grads is None or rec.grads[0] is None:
        return
    dy = rec.grads[0]
    ref_f, tol_f, ref_g, tol_g = gate_bwd(x, dy, c, ACT_NONE, x.dtype)
    C.within(f"{label}.dx", rec.res[0], torch.cat((ref_f, ref_g), 1), torch.cat((tol_f, tol_g), 1))
    C.equal(f"{label}.dres", rec.res[1], dy)


def _gemm64(a, w, K, bias=None):
    """(a w^T + bias, its bound (K + 2) U24 (|a| |w|^T + |bias|)) for an fp32 sum of K bf16 products and the bias."""
    ref, mag = a @ w.T, a.abs() @ w.abs().T
    if bias is not None:
        ref, mag = ref + bias, mag + bias.abs()
    return ref, (K + 2) * U24 * mag


def _check_slots(C, label, got, ref, bound, d):
    """A head in a slot: its d live columns within the bound, the slot's other columns +0.0."""
    C.within(label, got[:, :d], ref, bound)
    C.zero(label + "_pad", got[:, d:])


def attention_stage(C, name, layer, rec, params, geom):
    """The PixelSNAIL attention block (nn/modules.py `_attention_fwd` / `_attention_bwd` through `_AttentionPMFn`),
    sub-step by sub-step, each from its own recorded inputs (the Function's saved tensors, the recorded dy_b and the do,
    dq, dk, dv of ops.attn_bwd) and the parameters in their own shapes: one head of `key` q/k and `value` v channels in
    kernel slots (padded slot columns +0.0), q from the first C + 2 operand columns only (position and features: the
    image columns a wider q read meets must meet zero weights), k and v from C + 2 + c_img.
      forward   q, kv: GEMM bound and the bf16 store;  o, lse: tests/_attention_reference.attention with the table's
                strictness, SAFETY times its bounds (a strict row 0 is o = 0 and lse = 0 exactly);  y: the fp32
                projection of o;
      backward  dy_b: the bf16 cast of the incoming fp32 gradient, bit for bit;  do = dy_b Wp;  dq, dk, dv: the
                attention reference from the recorded do;  the six parameter gradients after unpack_grads: the weight
                gradients within the GEMM bound of their launch's split-K plan, the column sums within (P + 4) U24;
                da_kv: the fp32 sum of the kv and q dgrads, rounded to bf16 once, zero past C + 2 + c_img."""
    from pytorch_generative_b200 import ops

    label = f"attention {name}"
    A = layer.attn
    n, h, w = geom
    S = h * w
    cin, ckv, dk, dv = A.C + 2, A.C + 2 + A.c_img, A.key, A.value
    qs, vs = ops.head_slots(dk, dv)
    a_kv, q, kv, o, lse = rec.saved[:5]
    P = a_kv.shape[0]
    par = lambda k: params[f"{name}.{k}"].detach()
    wq, wkv, wp = (par(k).to(BF16).to(F64).reshape(par(k).shape[0], -1) for k in ("_q.weight", "_kv.weight",
                                                                                  "_proj.weight"))
    bq, bkv, bp = (par(k).to(F64) for k in ("_q.bias", "_kv.bias", "_proj.bias"))
    a = a_kv.to(F64)
    heads = lambda t, d: t[:, :d].reshape(n, S, 1, d).permute(0, 2, 1, 3)
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(P, -1)

    ref, err = _gemm64(a[:, :cin], wq, ops.round_up(cin, 8), bq)
    _check_slots(C, f"{label}.q", q, ref, _bf16_store(ref, err), dk)
    ref, err = _gemm64(a[:, :ckv], wkv, a_kv.shape[1], bkv)
    k, v = kv[:, :qs], kv[:, qs:]
    _check_slots(C, f"{label}.k", k, ref[:, :dk], _bf16_store(ref[:, :dk], err[:, :dk]), dk)
    _check_slots(C, f"{label}.v", v, ref[:, dk:], _bf16_store(ref[:, dk:], err[:, dk:]), dv)
    bwd = rec.grads is not None and rec.grads[0] is not None
    do = rec.attn["do"] if bwd else v
    at = attention(heads(q, dk), heads(k, dk), heads(v, dv), heads(do, dv), A.strict, dk, qs, vs, backward=bwd)
    _check_slots(C, f"{label}.o", o, flat(at["o"]), SAFETY * flat(at["b_o"]), dv)
    b_lse = SAFETY * at["b_lse"]
    if A.strict:
        b_lse[..., 0] = 0  # no visible key: lse is defined as 0
    C.within(f"{label}.lse", lse, at["lse"], b_lse)
    o64 = o[:, :dv].to(F64)
    ref, err = _gemm64(o64, wp, vs, bp)
    C.within(f"{label}.y", rec.out, ref, err)
    if not bwd:
        return

    dy, dy_b = rec.grads[0], rec.dy_b
    C.equal(f"{label}.dy_b", dy_b[:, :dv], dy.to(BF16))
    C.zero(f"{label}.dy_b_pad", dy_b[:, dv:])
    g = dy_b[:, :dv].to(F64)
    ref, err = _gemm64(g, wp.T, dv)
    _check_slots(C, f"{label}.do", do, ref, _bf16_store(ref, err), dv)
    d = {}
    for key, t, width in (("dq", rec.attn["dq"], dk), ("dk", rec.attn["dk"], dk), ("dv", rec.attn["dv"], dv)):
        _check_slots(C, f"{label}.{key}", t, flat(at[key]), SAFETY * flat(at["b_" + key]), width)
        d[key] = t[:, :width].to(F64)

    dwq_g, dbq_g, dwkv_g, dbkv_g, dwp_g, dbp_g = rec.res[1:7]
    dkv = torch.cat((d["dk"], d["dv"]), 1)
    # each weight gradient is one ops.linear_wgrad launch [m_out, n_out] over the P pixels, with the split-K factor
    # ops._split_k_for gives that launch: the bound of tests/_gemm_reference.py for that split
    for key, got, dyi, x, m_out, n_out in (("dw_q", dwq_g, d["dq"], a[:, :cin], qs, ops.round_up(cin, 8)),
                                           ("dw_kv", dwkv_g, dkv, a[:, :ckv], qs + vs, a_kv.shape[1]),
                                           ("dw_proj", dwp_g, g, o64, dy_b.shape[1], vs)):
        ref = dyi.T @ x
        err = gemm_bound(P, 1.0, dyi.abs().T @ x.abs(), torch.zeros_like(ref), ops._split_k_for(m_out, n_out, P))
        C.within(f"{label}.{key}", got.reshape(dyi.shape[1], -1), ref, err)
    for key, got, dyi in (("db_q", dbq_g, d["dq"]), ("db_kv", dbkv_g, dkv), ("db_proj", dbp_g, g)):
        C.within(f"{label}.{key}", got, dyi.sum(0), (P + 4) * U24 * dyi.abs().sum(0))
    ref, err = _gemm64(dkv, wkv.T, qs + vs)
    ref_q, err_q = _gemm64(d["dq"], wq.T, qs)
    ref[:, :cin] += ref_q
    err[:, :cin] += err_q + U24 * ref[:, :cin].abs()
    _check_slots(C, f"{label}.da_kv", rec.res[0], ref, _bf16_store(ref, err), ckv)


# ----------------------------------------------------------------------------------------------------------------------
# hand-offs between stages
# ----------------------------------------------------------------------------------------------------------------------
def out_dtype(T, name):
    """The dtype of what stage `name` hands on (its `value`)."""
    if name == "image":
        return F32
    layer = T[name]
    if layer.kind in ("act_cast", "gate") or layer.act in ("post", "pre_grad"):
        return BF16
    return F32 if layer.f32 else BF16


def _sum_bound(terms, dtype):
    """Bound of adding the terms in `dtype` (one rounding per addition) and storing the sum there."""
    u = U24 if dtype == F32 else U8
    return max(len(terms) - 1, 1) * u * sum(t.abs() for t in terms)


def _cols(got, ref):
    w = min(got.shape[1], ref.shape[1])
    return got[:, :w], ref[:, :w], got[:, w:]


def _attention_operand(C, name, layer, a_kv, features, image):
    """The attention operand [position | features | image | 0-pad]: bf16 of the reference's image_positional_encoding,
    the features' cast and bf16 of the image, each bit for bit, and +0.0 past them."""
    A = layer.attn
    pos = pm(image_positional_encoding(tuple(image.shape))).to(BF16).to(a_kv.device)
    c0 = 2 + A.C
    C.equal(f"attention {name}[position].a_kv", a_kv[:, :2], pos)
    C.equal(f"attention {name}[features].a_kv", a_kv[:, 2:c0], features[:, :A.C])
    C.equal(f"attention {name}[image].a_kv", a_kv[:, c0: c0 + A.c_img], pm(image).to(BF16))
    C.zero(f"attention {name}.a_kv_pad", a_kv[:, c0 + A.c_img:])


def forward_handoffs(C, T, values, inputs):
    """Each stage's recorded input against what the table says feeds it: bit for bit (dtype included) from one source,
    within one rounding in its dtype of the float64 sum of several; columns past the source's width must be +0.0.
    values: {stage: the tensor it hands on, "image": the model input}; inputs: {stage: its recorded input}."""
    for name, layer in T.items():
        if not layer.src or layer.src == ("image",) or name not in inputs:
            continue
        if layer.kind == "attention":
            _attention_operand(C, name, layer, inputs[name], values[layer.src[0]], values["image"])
            continue
        got, label = inputs[name], f"{layer.kind} {name}.x"
        srcs = [values[s] for s in layer.src]
        want = F32 if any(out_dtype(T, s) == F32 for s in layer.src) else BF16
        if got.dtype != want:
            C.failures[label] = f"{label}: the input is {got.dtype}, the table's sources give {want}"
            C.ratios[label] = float("inf")
            continue
        if len(srcs) == 1:
            g, r, extra = _cols(got, srcs[0])
            C.equal(label, g, r)
        else:
            w = min(s.shape[1] for s in srcs)
            terms = [s[:, :w].to(F64) for s in srcs]
            g, extra = got[:, :w], got[:, w:]
            C.within(label, g, sum(terms), _sum_bound(terms, want))
        C.zero(f"{layer.kind} {name}.x_pad", extra)


def backward_handoffs(C, T, incoming, returned):
    """A stage output with several consumers receives the sum autograd forms in the output's dtype of the gradients its
    consumers returned for it: within one rounding per addition of their float64 sum; one with a single consumer
    receives what that consumer returned, in the output's dtype, bit for bit.  incoming: {stage: the gradient its
    backward received}; returned: {(consumer, source or 'res'): the gradient the consumer returned for that input, None
    if it returned none}, for the consumers whose backward ran (the last layer's v and h streams reach no loss).  A
    consumer that ran and returned no gradient fails the check."""
    consumers = {}
    for name, layer in T.items():
        for s in layer.src or ():
            consumers.setdefault(s, []).append((name, s))
        if layer.res and layer.res_of == "out":
            consumers.setdefault(layer.res, []).append((name, "res"))
    for name, cons in consumers.items():
        if name == "image" or incoming.get(name) is None:
            continue
        label = f"{T[name].kind} {name}.dy"
        got, dtype = incoming[name], out_dtype(T, name)
        terms = []
        for key in cons:
            if key not in returned:  # a consumer whose own output reached no loss (the last layer's v and h streams)
                continue
            t = returned[key]
            if t is None:
                C.failures[label] = f"{label}: consumer {key[0]} returned no gradient for it"
                C.ratios[label] = float("inf")
                break
            terms.append(t.to(dtype).to(F64))  # a sum's backward hands its gradient on in each summand's dtype
        else:
            if not terms:
                continue
            w = min([got.shape[1]] + [t.shape[1] for t in terms])
            if len(cons) == 1:
                C.equal(label, got[:, :w], returned[cons[0]].to(dtype)[:, :w])
                continue
            terms = [t[:, :w] for t in terms]
            C.within(label, got[:, :w], sum(terms), _sum_bound(terms, dtype))


# ----------------------------------------------------------------------------------------------------------------------
# the GatedPixelCNN and PixelSNAIL chain: the stage references composed along the graph, in float64
# ----------------------------------------------------------------------------------------------------------------------
def masked(layer, w):
    """The weight a stage reads: a mask-centre causal convolution's times the reference's causal_mask."""
    if not layer.mask:
        return w
    return w * causal_mask(*w.shape[2:], True).to(w)


def graph_chain(T, P, x):
    """The logits of the stage graph T in float64: each stage reads the sum of its sources' outputs (`stage_out`), a
    residual the output of the stage the table names.  P: parameters by name."""
    values = {"image": x}
    for name, layer in T.items():
        xin = sum(values[s] for s in layer.src)
        if layer.kind in ("conv", "image"):
            res = values[layer.res] if layer.res else None
            w = P[name + ".weight"]
            w = w + (masked(layer, w) - w).detach()  # the reference masks outside autograd: dw stays dense
            y = stage_y(layer, stage_in(layer, xin), w, P[name + ".bias"], res)
            values[name] = stage_out(layer, y)
        elif layer.kind == "gate":
            values[name] = gated_activation(xin)
        elif layer.kind == "gated_res":
            values[name] = values[layer.res] + gated_activation(xin, lambda z: z)
        elif layer.kind == "attention":
            A = layer.attn
            pos = image_positional_encoding(tuple(x.shape)).to(x)
            values[name] = causal_attention(torch.cat((pos, xin), 1), P, name + ".", 1, A.key, A.value, A.strict, x)
        else:
            assert layer.kind in ("act_cast", "stream"), layer.kind
            values[name] = xin
    return values[name]
