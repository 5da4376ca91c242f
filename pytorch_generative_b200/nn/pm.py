"""Pixel-major functional ops with autograd: the building blocks of the conv-model stacks and of the drop-in Modules.

The model stacks (`models/gated_pixel_cnn.py`, `models/pixel_snail.py`) keep every activation pixel-major between the
image-channel input layer and the logits: `[P = N*H*W, C]` matrices, bf16 where the tensor is only ever a tensor-core
operand, fp32 for residual streams.  The drop-in Modules (`CausalConv2d`, `TapConv2d`, `GatedActivation`) take and
return NCHW fp32 like the reference: each is `to_pm`, one op of this file and `from_pm`.  Each function here is one
`torch.autograd.Function` over such matrices whose forward / backward are the C-ABI kernels:

  * `conv`      any stride-1 convolution with an input-sized output, at any geometry, with up to 225 kernel positions
                (e.g. 15 x 15) and any dilation.  A 1x1 conv is one GEMM.  Wider kernels run as a tap loop on the wgmma GEMM
                (`pg_gemm_bf16_conv_taps`: the shifted input is read in place through 4-D TMA boxes) where the image,
                both channel widths and the tap offsets suit it (`L.conv_gemm_supported`),
                else as `pg_tap_gather` -> GEMM, with `pg_tap_scatter` folding the input gradient back.  The bias, a
                residual and the NEXT layer's input activation are fused into the epilogue; the input gradient carries
                the derivative of THIS layer's input activation;
  * `image_conv` an NCHW tensor (the image) straight to pixel-major: the direct fp32 kernel `small_conv` for
                contractions as short as an image-channel layer's (`tapconv.small_conv_ok`), else `conv`;
  * `gated`     GatedActivation; `act_cast` materialises act(x) in bf16 where no producer epilogue could.

Reference call sites: gated_pixel_cnn.py:112-130, pixel_snail.py:27-28,52-56,112-119, nn/convolution.py:41-43,62-66.
"""

import collections

import torch

from .. import _lib as L
from .. import ops
from .tapconv import conv_taps, small_conv_ok

F32, BF16 = torch.float32, torch.bfloat16
Geom = collections.namedtuple("Geom", "n h w")


# --------------------------------------------------------------------------------------------------
# layout boundary
# --------------------------------------------------------------------------------------------------
class _FromPM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x_pm, geom, c, act):
        ctx.width, ctx.c, ctx.act = x_pm.shape[1], c, act
        ctx.save_for_backward(x_pm if act != L.ACT_NONE else None)
        return ops.pm_to_nchw(x_pm, geom.n, c, geom.h, geom.w, act=act)

    @staticmethod
    def backward(ctx, dy):
        if ctx.act == L.ACT_NONE:
            return ops.nchw_to_pm(dy, F32, width=ctx.width), None, None, None
        (pre,) = ctx.saved_tensors
        c = ctx.c
        d = ops.nchw_to_pm(dy, BF16, width=ctx.width)
        L.dact_mul(d[:, :c], pre[:, :c], ctx.act, d[:, :c])
        return d, None, None, None


def from_pm(x_pm, geom, c, act=L.ACT_NONE):
    """act([P, >=c] fp32 pixel-major) -> [N, c, H, W] fp32.  With an activation its derivative is taken at the saved
    fp32 pre-activation, and the gradient leaves in bf16: the GEMM operand the producing convolution reads."""
    return _FromPM.apply(x_pm, geom, c, act)


class _ToPM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dtype, width):
        ctx.shape = x.shape
        return ops.nchw_to_pm(x, dtype, width=width)

    @staticmethod
    def backward(ctx, dy):
        n, c, h, w = ctx.shape
        return ops.pm_to_nchw(dy.float().contiguous(), n, c, h, w), None, None


def to_pm(x, dtype, width=None):
    """[N, C, H, W] fp32 -> [P, width >= C] pixel-major in `dtype` (extra columns zero)."""
    return _ToPM.apply(x, dtype, width)


# --------------------------------------------------------------------------------------------------
# elementwise
# --------------------------------------------------------------------------------------------------
class _ActCast(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, act):
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
        L.act_cast(x, act, out)
        ctx.act = act
        ctx.save_for_backward(out if act != L.ACT_NONE else None)
        ctx.in_dtype = x.dtype
        return out

    @staticmethod
    def backward(ctx, dy):
        (out,) = ctx.saved_tensors
        if ctx.act == L.ACT_NONE:
            return dy.to(ctx.in_dtype), None
        # act' from the activated value (relu / elu): torch elementwise on a [P, C] matrix, off the hot path (the
        # stacks take the fused route: the consumer's dgrad epilogue applies the derivative)
        a = out.float()
        d = (a > 0).float() if ctx.act == L.ACT_RELU else torch.where(a > 0, torch.ones_like(a), a + 1)
        return (dy.float() * d).to(ctx.in_dtype), None


def act_cast(x, act=L.ACT_NONE):
    """bf16(act(x)) of a pixel-major matrix (fp32 or bf16)."""
    if act == L.ACT_NONE and x.dtype == BF16:
        return x
    return _ActCast.apply(x, act)


class _Gated(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, act, dtype):
        P, c2 = x.shape
        y = torch.empty(P, c2 // 2, dtype=dtype, device=x.device)
        L.gated_act_fwd(x, y, act)
        ctx.save_for_backward(x)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dyc = dy.contiguous()
        if dyc.dtype != x.dtype:
            dyc = dyc.to(x.dtype)
        dx = torch.empty_like(x)
        L.gated_act_bwd(x, dyc, dx, ctx.act)
        return dx, None, None


def gated(x, act, dtype=BF16):
    """act(x[:, :C]) * sigmoid(x[:, C:]) -> [P, C] in `dtype` (reference nn/convolution.py:62-66), any C."""
    return _Gated.apply(x.contiguous(), act, dtype)


class _GatedRes(torch.autograd.Function):
    """res + gate(x) in one pass (fp32 stream in / out); backward: d res = dy, d x = gate'(x) dy."""

    @staticmethod
    def forward(ctx, x, res, act):
        y = torch.empty_like(res)
        L.gated_res_fwd(x, res, y, act)
        ctx.save_for_backward(x)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        L.gated_act_bwd(x, dy, dx, ctx.act)  # fp32 dy over a bf16 x is a supported combination
        return dx, dy, None


def gated_res(x, res, act):
    """res + act(x[:, :C]) * sigmoid(x[:, C:]) -> fp32 [P, C]: a gated residual block's output stream, any C."""
    return _GatedRes.apply(x.contiguous(), res.contiguous(), act)


# --------------------------------------------------------------------------------------------------
# convolutions
# --------------------------------------------------------------------------------------------------
class _SmallConv(torch.autograd.Function):
    """Direct fp32 convolution (Cin*kh*kw <= 160) of pre_act(x): NCHW fp32 in, pixel-major fp32 out."""

    @staticmethod
    def forward(ctx, x, weight, bias, padding, pre_act, dilation):
        x = x.contiguous().float()
        n, _, h, w = x.shape
        cout = weight.shape[0]
        out = torch.empty(n * h * w, cout, dtype=F32, device=x.device)
        L.conv_small_fwd(x, weight.detach().contiguous(), None if bias is None else bias.detach(), padding, out_f32=out,
                         pre_act=pre_act, dilation=dilation)
        ctx.save_for_backward(x, weight)
        ctx.padding, ctx.has_bias, ctx.pre_act, ctx.dilation = padding, bias is not None, pre_act, dilation
        return out

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous().float()
        dw = torch.zeros_like(weight)
        db = torch.zeros(weight.shape[0], dtype=F32, device=dy.device) if ctx.has_bias else None
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        L.conv_small_bwd(x, weight.detach().contiguous(), dy, ctx.padding, dw=dw, dbias=db, dx=dx, pre_act=ctx.pre_act,
                         dilation=ctx.dilation)
        return dx, dw, db, None, None, None


def small_conv(x_nchw, weight, bias, padding, pre_act=L.ACT_NONE, dilation=(1, 1)):
    return _SmallConv.apply(x_nchw, weight, bias, tuple(padding), pre_act, tuple(dilation))


def _check_padding(weight, padding, dilation=(1, 1)):
    """The padded output of a kh x kw kernel with dilation d covers the input when 2 pad >= d (k - 1) on both axes."""
    kh, kw = weight.shape[-2:]
    if 2 * padding[0] < dilation[0] * (kh - 1) or 2 * padding[1] < dilation[1] * (kw - 1):
        raise NotImplementedError(f"conv: padding {tuple(padding)} is too small for an input-sized output of a {kh}x{kw} "
                                  f"kernel with dilation {tuple(dilation)} (not a shape on the path)")


def image_conv(x_nchw, weight, bias, padding, pre_act=L.ACT_NONE, dilation=(1, 1)):
    """conv2d(pre_act(x), weight, bias, padding, dilation) cropped to x's H x W: NCHW fp32 in, fp32 pixel-major
    [P, Cout] out.  A contraction this short (image-channel inputs, 16/32-channel layers) is not tensor-core work: the
    direct fp32 kernel, exact to 1e-3 (no bf16 rounding of the operands); a longer one runs through `conv`."""
    if small_conv_ok(weight.shape):
        _check_padding(weight, padding, dilation)
        return small_conv(x_nchw, weight, bias, padding, pre_act, dilation)
    n, c, h, w = x_nchw.shape
    y, _ = conv(to_pm(x_nchw, F32, ops.round_up(c, 8)), weight, bias, Geom(n, h, w), padding, in_act=pre_act,
                out_f32=True, dilation=dilation)
    return y


COMPANION, PRE_GRAD, POST = 0, 1, 2  # what the activated output `ya` of a conv is to autograd (see `conv`)
POINTWISE, TAP_LOOP, GATHER = 0, 1, 2  # how `_Conv` computes a convolution; picked per call from the geometry
# GELU's derivative does not follow from its output, so a GELU operand travels with its derivative: a = bf16(GELU(x)),
# d = bf16(GELU'(x)), both [P, Cin_p] with one pitch (a's pad columns zero).  The consumer's dgrad applies d as given.
GeluOperand = collections.namedtuple("GeluOperand", "a d")


def gelu_operand(x, width=None):
    """GeluOperand of an fp32 pixel-major matrix x [P, C] (pg_gelu_cast): for values no epilogue produces."""
    width = width or ops.round_up(x.shape[1], 8)
    a = torch.empty(x.shape[0], width, dtype=BF16, device=x.device)
    d = torch.empty_like(a)
    L.gelu_cast(x.detach(), a, d)
    return GeluOperand(a, d)


class _Conv(torch.autograd.Function):
    """y = conv(xa) + bias (+ res), xa = bf16(in_act(x)) given by the caller.  Returns (y, ya): y fp32 / bf16 / None,
    ya = bf16(emit(y)) or None; with a GELU emit that is not POST, (y, ya, bf16(GELU'(y))).  xd: bf16(in_act'(x)) for
    an input activation whose derivative does not follow from its output (GELU), applied as given by the dgrad."""

    @staticmethod
    def forward(ctx, x, xa, weight, bias, res, geom, taps, in_act, emit, emit_mode, out_f32, want_main, xd=None):
        cout = weight.shape[0]
        cin_p = xa.shape[1]
        if len(taps) == 1 and taps[0] == (0, 0):
            mode = POINTWISE
        elif L.conv_gemm_supported(geom.h, geom.w, cin_p, taps) and L.conv_gemm_supported(geom.h, geom.w, cout, taps):
            mode = TAP_LOOP  # the dgrad reads dy through TMA as well
        else:
            mode = GATHER
        wcat = ops.pack_taps(weight, cin_p)
        b = None if bias is None else bias.detach()
        want_act = emit is not None
        # a GELU emit that a consumer reads as its input also stores GELU' (the derivative that consumer applies)
        gelu2 = emit == L.ACT_GELU and emit_mode != POST
        kw_out = dict(act=emit if want_act else L.ACT_NONE, res0=res, want_bf16=want_act,
                      want_pre=gelu2 or (want_main and not out_f32), want_f32=want_main and out_f32, pre_deriv=gelu2)
        a = xa  # the GEMM operand: xa itself, or its taps side by side
        if mode == GATHER:
            a = torch.empty(xa.shape[0], len(taps) * cin_p, dtype=BF16, device=xa.device)
            L.tap_gather(xa, geom.n, geom.h, geom.w, cin_p, taps, L.ACT_NONE, a)  # xa is activated already
        if mode == TAP_LOOP:
            ya, yb, yf = ops.conv_fwd(xa, wcat, b, geom.n, geom.h, geom.w, taps, **kw_out)
        else:
            ya, yb, yf = ops.linear_fwd(a, wcat, b, **kw_out)
        # backward needs the operand itself (wgrad); the activated input also yields in_act' (dgrad epilogue), the
        # activated output yields emit' when it is a true post-activation output
        # undefined output gradients arrive as None, not as zero tensors: the companion output is never differentiated, and
        # a materialised zero gradient for it costs a fill, a dtype conversion and an add per layer
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(xa, a, wcat, ya if (want_act and emit_mode == POST and emit != L.ACT_NONE) else None, xd)
        ctx.meta = (geom, taps, mode, in_act, weight.shape, bias is not None, None if res is None else res.dtype,
                    x.dtype, emit, emit_mode)
        y = (yf if out_f32 else yb) if want_main else None
        ctx.n_inputs = 12 if xd is None else 13
        if ya is not None and emit_mode == COMPANION:
            ctx.mark_non_differentiable(ya)
        if gelu2:  # the third output: GELU'(y), stored by the same epilogue (yb)
            ctx.mark_non_differentiable(yb)
            return y, ya, yb
        return y, ya

    @staticmethod
    def backward(ctx, dy, dya, *_):
        xa, a, wcat, ya, xd = ctx.saved_tensors
        geom, taps, mode, in_act, wshape, has_bias, res_dtype, x_dtype, emit, emit_mode = ctx.meta
        cout, cin, kh, kw = wshape
        cin_p = xa.shape[1]
        cout_p = ops.round_up(cout, 8)
        T = len(taps)
        if dy is None and dya is None:  # nothing downstream used this convolution
            return (None,) * ctx.n_inputs
        if emit_mode == COMPANION:
            dya = None
        if dya is not None and emit_mode == POST and emit != L.ACT_NONE:
            # gradient w.r.t. the activated output: back through emit (relu / elu) from the activated value itself
            d = torch.empty(ya.shape, dtype=BF16, device=ya.device)
            L.dact_from_out(dya.contiguous(), ya, emit, d)
            dya = d
        if dy is None:
            dy = dya
        elif dya is not None:
            dy = dy + dya.to(dy.dtype)
        dy = dy.contiguous()
        if dy.dtype == BF16 and cout_p == cout:
            dyb = dy
        elif cout_p == cout:
            dyb = torch.empty(dy.shape, dtype=BF16, device=dy.device)
            L.act_cast(dy, L.ACT_NONE, dyb)
        else:  # a handful of output channels (the logits): pad the operand to the 16-byte TMA pitch
            dyb = torch.zeros(dy.shape[0], cout_p, dtype=BF16, device=dy.device)
            dyb[:, :cout] = dy
        db = dw = None
        if ctx.needs_input_grad[2]:
            # weight and bias gradient in one launch: the wgrad GEMM reduces the dy tiles it stages (ops.linear_wgrad)
            dwcat = torch.zeros(cout_p, T * cin_p, dtype=F32, device=dy.device)
            dbp = torch.zeros(cout_p, dtype=F32, device=dy.device) if has_bias else None
            if mode == TAP_LOOP:
                ops.conv_wgrad(dyb, xa, dwcat, geom.n, geom.h, geom.w, taps, db_out=dbp)
            else:
                ops.linear_wgrad(dyb, a, dwcat, db_out=dbp)
            dw = dwcat[:cout].view(cout, kh, kw, cin_p)[..., :cin].permute(0, 3, 1, 2).contiguous()
            db = dbp[:cout] if has_bias else None
        elif has_bias:
            db = ops.bias_grad(dyb[:, :cout])
        dx = None
        if ctx.needs_input_grad[0]:
            want_f32 = x_dtype == F32
            if xd is not None:  # the derivative came with the operand (GELU)
                dact, aux = L.ACT_GIVEN, xd
            else:
                dact = L.DACT_FROM_OUT.get(in_act, L.ACT_NONE)
                aux = xa if dact != L.ACT_NONE else None
            if mode == POINTWISE:
                r = ops.linear_dgrad(dyb[:, :cout], wcat, aux=aux, dact=dact, want_f32=want_f32)
                dx = r[1] if want_f32 else r
            elif mode == TAP_LOOP:
                dxb, dxf = ops.conv_dgrad(dyb, wcat, cin_p, geom.n, geom.h, geom.w, taps, aux=aux, dact=dact,
                                          want_f32=want_f32, want_bf16=not want_f32)
                dx = dxf if want_f32 else dxb
            else:  # dX_cat, then each tap's slice folded back onto the pixel it was read from
                dx = torch.empty(xa.shape, dtype=x_dtype, device=dy.device)
                L.tap_scatter(ops.linear_dgrad(dyb[:, :cout], wcat), geom.n, geom.h, geom.w, cin_p, taps, dact, aux,
                              dx_f32=dx if want_f32 else None, dx_bf16=None if want_f32 else dx)
        dres = None
        if res_dtype is not None:  # d(res) = dy: hand over the copy that already has the residual's dtype
            dres = dy if dy.dtype == res_dtype else (dyb if (res_dtype == BF16 and cout_p == cout) else dy.to(res_dtype))
        return (dx, None, dw, db, dres, None, None, None, None, None, None, None, None)[: ctx.n_inputs]


def conv(x, weight, bias, geom, padding=(0, 0), *, in_act=L.ACT_NONE, xa=None, res=None, emit=None, emit_mode=COMPANION,
         out_f32=False, want_main=True, dilation=(1, 1)):
    """Convolution of a pixel-major activation.

    x        [P, Cin_p] differentiable input (bf16, or an fp32 residual stream), BEFORE its input activation; an input
             narrower than a multiple of 8 columns is zero-padded to one (the 16-byte operand pitch);
    in_act   activation the reference applies in front of this conv (ReLU / ELU / none); its derivative is applied by
             this conv's dgrad, so the gradient this op returns for x is w.r.t. the PRE-activation value;
    xa       bf16(in_act(x)) if a producer epilogue already emitted it (else built here with one elementwise pass);
    res      optional [P, Cout] added to the output in the epilogue: fp32 (a residual / skip stream) or bf16 (a short-lived
             sum such as GatedPixelCNN's vertical-to-horizontal link; its gradient then stays bf16 as well);
    emit     activation id (or ACT_NONE for a plain bf16 copy) of a second, bf16 output produced by the same epilogue;
    emit_mode COMPANION: `ya` is a non-differentiable operand copy of y (pass it as `xa` to the consumers of y);
             PRE_GRAD: `ya` stands for y in the graph and may only feed `conv(ya, in_act=emit, xa=ya)`, whose fused
             derivative makes the gradient it receives the gradient w.r.t. y (use with want_main=False: the
             pre-activation tensor is then never written);  POST: `ya` is an ordinary activated output;
             with emit=GELU (COMPANION or PRE_GRAD) `ya` is a GeluOperand: the epilogue also stores GELU'(y), so the
             main output, if wanted, must be fp32 (in PRE_GRAD feed `ya.a` as x);
    GELU     in_act=GELU takes `xa` as a GeluOperand (built by pg_gelu_cast when None); the dgrad multiplies by its
             stored derivative (ACT_GIVEN) in every mode;
    out_f32  the main output is fp32 (a stream) instead of bf16;
    dilation nn.Conv2d's dilation: kernel position (i, j) is the tap (i d_h - pad_h, j d_w - pad_w).
    Returns (y, ya)."""
    kh, kw = weight.shape[-2:]
    _check_padding(weight, padding, dilation)
    taps = conv_taps(kh, kw, padding[0], padding[1], dilation[0], dilation[1])
    if len(taps) > L.MAX_TAPS:
        raise NotImplementedError(f"conv: {len(taps)} taps exceed the {L.MAX_TAPS} of the tap kernels (kernel {kh}x{kw}; "
                                  f"at most {L.MAX_TAPS} kernel positions, e.g. 15 x 15)")
    if emit == L.ACT_GELU and emit_mode != POST and want_main and not out_f32:
        raise NotImplementedError("conv: a GELU emit stores GELU' where a bf16 main output would go; ask for out_f32")
    if in_act == L.ACT_GELU:
        return _gelu_input_conv(x, weight, bias, geom, taps, xa, res, emit, emit_mode, out_f32, want_main)
    if in_act != L.ACT_NONE and in_act not in L.DACT_FROM_OUT:
        raise NotImplementedError(f"conv: input activation {in_act} has no derivative from its output (ReLU / ELU do)")
    if x.shape[1] % 8:
        same = xa is x
        x = torch.nn.functional.pad(x, (0, -x.shape[1] % 8))
        xa = x if same else None
    if xa is None:
        xa = act_cast(x, in_act) if (in_act != L.ACT_NONE or x.dtype != BF16) else x
    return _pack_gelu(_Conv.apply(x, xa.detach() if xa is not x else xa, weight, bias, res, geom, taps, in_act, emit,
                                  emit_mode, out_f32, want_main))


def _gelu_input_conv(x, weight, bias, geom, taps, xa, res, emit, emit_mode, out_f32, want_main):
    """`conv` with in_act=GELU: xa is a GeluOperand, or None to build one from the fp32 x."""
    width = ops.round_up(x.shape[1], 8)
    same = xa is not None and xa.a is x  # PRE_GRAD: the producer's GELU(y) stands for y
    pad = lambda t: torch.nn.functional.pad(t, (0, width - t.shape[1]))
    if x.shape[1] != width:
        x = pad(x)
    if same:
        xa = GeluOperand(x, xa.d if xa.d.shape[1] == width else pad(xa.d))
    elif xa is None:
        if x.dtype != F32:
            raise NotImplementedError("conv: a GELU input without its GeluOperand must be an fp32 stream")
        xa = gelu_operand(x, width)
    elif xa.a.shape[1] != width:
        xa = GeluOperand(pad(xa.a.detach()), pad(xa.d))
    out = _Conv.apply(x, xa.a if same else xa.a.detach(), weight, bias, res, geom, taps, L.ACT_GELU, emit, emit_mode,
                      out_f32, want_main, xa.d.detach())
    return _pack_gelu(out)


def _pack_gelu(out):
    """(y, ya) of a `_Conv` call; a GELU emit's (ya, GELU'(y)) becomes one GeluOperand."""
    return (out[0], GeluOperand(out[1], out[2])) if len(out) == 3 else out


# --------------------------------------------------------------------------------------------------
# strided and transposed convolutions (reference models/vae/vaes.py Encoder / Decoder)
# --------------------------------------------------------------------------------------------------
def conv_out_size(size, k, stride, pad):
    """nn.Conv2d's output side (dilation 1)."""
    return (size + 2 * pad - k) // stride + 1


def conv_t_out_size(size, k, stride, pad):
    """nn.ConvTranspose2d's output side (dilation 1, output_padding 0)."""
    return (size - 1) * stride - 2 * pad + k


def _strided_spec(conv):
    """(taps, stride) of an nn.Conv2d / nn.ConvTranspose2d holder; NotImplementedError for the settings the strided
    kernels do not compute: groups, dilation, output_padding, a padding mode other than zeros, a string padding,
    unequal strides or more than MAX_TAPS kernel positions."""
    who = type(conv).__name__
    transposed = isinstance(conv, torch.nn.ConvTranspose2d)
    out_pad = tuple(conv.output_padding) if transposed else (0, 0)
    if (conv.groups != 1 or tuple(conv.dilation) != (1, 1) or out_pad != (0, 0) or conv.padding_mode != "zeros"
            or isinstance(conv.padding, str)):
        raise NotImplementedError(f"{who}: only groups 1, dilation 1, output_padding 0 and explicit zero padding are on "
                                  f"the strided path (got groups {conv.groups}, dilation {tuple(conv.dilation)}, "
                                  f"output_padding {out_pad}, padding {conv.padding!r}, mode {conv.padding_mode!r})")
    kh, kw = conv.kernel_size
    if kh * kw > L.MAX_TAPS:
        raise NotImplementedError(f"{who}: a {kh}x{kw} kernel exceeds the {L.MAX_TAPS} taps of the strided kernels")
    if conv.stride[0] != conv.stride[1]:
        raise NotImplementedError(f"{who}: stride {tuple(conv.stride)}: only equal strides are on the strided path")
    return conv_taps(kh, kw, conv.padding[0], conv.padding[1]), conv.stride[0]


def strided_geom(conv, geom):
    """Geometry of the output of an nn.Conv2d / nn.ConvTranspose2d holder on a `geom` input, as torch sizes it;
    ValueError, before any launch, when it would be empty."""
    _strided_spec(conv)
    size = conv_t_out_size if isinstance(conv, torch.nn.ConvTranspose2d) else conv_out_size
    (kh, kw), s, (ph, pw) = conv.kernel_size, conv.stride[0], conv.padding
    ho, wo = size(geom.h, kh, s, ph), size(geom.w, kw, s, pw)
    if ho < 1 or wo < 1:
        raise ValueError(f"{type(conv).__name__}: a {geom.h}x{geom.w} input is too small for a {kh}x{kw} kernel at "
                         f"stride {s} and padding {tuple(conv.padding)}")
    return Geom(geom.n, ho, wo)


def _operand(x, in_act):
    """(x padded to a multiple of 8 columns with zeros, bf16(in_act(x)))."""
    if x.shape[1] % 8:
        x = torch.nn.functional.pad(x, (0, -x.shape[1] % 8))
    xa = act_cast(x, in_act) if (in_act != L.ACT_NONE or x.dtype != BF16) else x
    return x, xa


def _grad_operand(dy, y_act, emit, cout_p):
    """bf16 [P, cout_p] GEMM operand of the output gradient; through emit' (from the activated output) when the output
    was emit(y)."""
    dy = dy.contiguous()
    if emit is not None and emit != L.ACT_NONE:
        d = torch.empty(y_act.shape, dtype=BF16, device=dy.device)
        L.dact_from_out(dy, y_act, emit, d)
        return d
    if dy.dtype == BF16:
        return dy
    d = torch.empty(dy.shape, dtype=BF16, device=dy.device)
    L.act_cast(dy, L.ACT_NONE, d)
    return d


class _StridedConv(torch.autograd.Function):
    """y = conv2d(xa, weight, bias, stride, padding) on pixel-major matrices: pg_strided_gather -> GEMM.  Returns bf16
    emit(y) (an ordinary activated output) when emit is set, else y (fp32 when out_f32, else bf16); [P_out, cout_p]
    with exactly zero pad columns."""

    @staticmethod
    def forward(ctx, x, xa, weight, bias, rows, spatial, taps, stride, in_act, emit, out_f32):
        cout = weight.shape[0]
        cout_p = ops.round_up(cout, 8)
        cin_p = xa.shape[1]
        wcat = ops.pack_taps(weight, cin_p, cout_p=cout_p)
        a = torch.empty(rows[0] * rows[1] * rows[2], len(taps) * cin_p, dtype=BF16, device=xa.device)
        L.strided_gather(xa, rows, spatial, cin_p, taps, stride, a)
        b = None if bias is None else ops.padded_bias(bias, cout_p)
        act = L.ACT_NONE if emit is None else emit
        yb, _, yf = ops.linear_fwd(a, wcat, b, act=act, want_bf16=emit is not None or not out_f32,
                                   want_f32=emit is None and out_f32)
        y = yf if yf is not None else yb
        ctx.save_for_backward(xa, a, wcat, y if emit not in (None, L.ACT_NONE) else None)
        ctx.meta = (rows, spatial, taps, stride, in_act, emit, weight.shape, bias is not None, x.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xa, a, wcat, ya = ctx.saved_tensors
        rows, spatial, taps, stride, in_act, emit, wshape, has_bias, x_dtype = ctx.meta
        cout, cin, kh, kw = wshape
        cout_p, cin_p = wcat.shape[0], xa.shape[1]
        dyb = _grad_operand(dy, ya, emit, cout_p)
        dw = db = dx = None
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
            # weight and bias gradient in one launch: the wgrad GEMM reduces the dy tiles it stages
            dwcat = torch.zeros(cout_p, wcat.shape[1], dtype=F32, device=dyb.device)
            dbp = torch.zeros(cout_p, dtype=F32, device=dyb.device) if has_bias else None
            ops.linear_wgrad(dyb, a, dwcat, db_out=dbp)
            dw = dwcat[:cout].view(cout, kh, kw, cin_p)[..., :cin].permute(0, 3, 1, 2).contiguous()
            db = dbp[:cout] if has_bias else None
        if ctx.needs_input_grad[0]:
            dact = L.DACT_FROM_OUT.get(in_act, L.ACT_NONE)
            dx = torch.empty(xa.shape, dtype=x_dtype, device=dyb.device)
            f32 = x_dtype == F32
            L.strided_scatter(ops.linear_dgrad(dyb, wcat), rows, spatial, cin_p, taps, stride, dact=dact,
                              x_pre=xa if dact != L.ACT_NONE else None, out_f32=dx if f32 else None,
                              out_bf16=None if f32 else dx)
        return dx, None, dw, db, None, None, None, None, None, None, None


def conv_strided(x, conv, geom, *, in_act=L.ACT_NONE, emit=None, out_f32=False):
    """`conv` (an nn.Conv2d: its weight, bias, stride and padding) of a pixel-major activation x [N*H*W, Cin(_p)]
    (bf16, or an fp32 stream), BEFORE its input activation `in_act` (whose derivative the input gradient carries, as in
    `conv`).  Output sizes follow nn.Conv2d.  Returns (y [N*Ho*Wo, round_up(Cout, 8)], Geom(N, Ho, Wo)): bf16 emit(y)
    when `emit` is set (its gradient goes back through emit' from the activated value), else y in fp32 (out_f32) or
    bf16."""
    taps, stride = _strided_spec(conv)
    out_geom = strided_geom(conv, geom)
    if in_act != L.ACT_NONE and in_act not in L.DACT_FROM_OUT:
        raise NotImplementedError(f"conv_strided: input activation {in_act} has no derivative from its output")
    x, xa = _operand(x, in_act)
    y = _StridedConv.apply(x, xa.detach() if xa is not x else xa, conv.weight, conv.bias, tuple(out_geom), tuple(geom),
                           taps, stride, in_act, emit, out_f32)
    return y, out_geom


class _TransposedConv(torch.autograd.Function):
    """y = conv_transpose2d(xa, weight, bias, stride, padding): GEMM X W_t^T into fp32 Y_cat, then pg_strided_scatter
    adds the bias and writes y (fp32) or emit(y) (bf16).  [P_out, cout_p] with exactly zero pad columns."""

    @staticmethod
    def forward(ctx, x, xa, weight, bias, rows, spatial, taps, stride, in_act, emit, out_f32):
        cout = weight.shape[1]
        cout_p = ops.round_up(cout, 8)
        cin_p = xa.shape[1]
        wt = ops.pack_taps_t(weight, cin_p, cout_p)
        _, _, ycat = ops.linear_fwd(xa, wt, want_bf16=False, want_f32=True)
        p_out = spatial[0] * spatial[1] * spatial[2]
        want_bf16 = emit is not None or not out_f32
        yf = torch.empty(p_out, cout_p, dtype=F32, device=xa.device) if not want_bf16 else None
        yb = torch.empty(p_out, cout_p, dtype=BF16, device=xa.device) if want_bf16 else None
        L.strided_scatter(ycat, rows, spatial, cout_p, taps, stride, bias=None if bias is None else bias.detach(),
                          act=L.ACT_NONE if emit is None else emit, out_f32=yf, out_bf16=yb)
        y = yb if want_bf16 else yf
        ctx.save_for_backward(xa, wt, y if emit not in (None, L.ACT_NONE) else None)
        ctx.meta = (rows, spatial, taps, stride, in_act, emit, weight.shape, bias is not None, x.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xa, wt, ya = ctx.saved_tensors
        rows, spatial, taps, stride, in_act, emit, wshape, has_bias, x_dtype = ctx.meta
        cin, cout, kh, kw = wshape
        cin_p = xa.shape[1]
        cout_p = wt.shape[0] // len(taps)
        dyb = _grad_operand(dy, ya, emit, cout_p)
        dycat = torch.empty(xa.shape[0], wt.shape[0], dtype=BF16, device=dyb.device)
        L.strided_gather(dyb, rows, spatial, cout_p, taps, stride, dycat)
        dw = db = dx = None
        if ctx.needs_input_grad[2]:
            dwt = torch.zeros(wt.shape, dtype=F32, device=dyb.device)
            ops.linear_wgrad(dycat, xa, dwt)
            dw = dwt.view(kh, kw, cout_p, cin_p)[:, :, :cout, :cin].permute(3, 2, 0, 1).contiguous()
        if has_bias and ctx.needs_input_grad[3]:
            db = ops.bias_grad(dyb[:, :cout])  # fixed-order column sums: the GEMMs only see dY_cat
        if ctx.needs_input_grad[0]:
            dact = L.DACT_FROM_OUT.get(in_act, L.ACT_NONE)
            r = ops.linear_dgrad(dycat, wt, aux=xa if dact != L.ACT_NONE else None, dact=dact, want_f32=x_dtype == F32)
            dx = r[1] if x_dtype == F32 else r
        return dx, None, dw, db, None, None, None, None, None, None, None


def conv_transposed(x, conv, geom, *, in_act=L.ACT_NONE, emit=None, out_f32=False):
    """`conv` (an nn.ConvTranspose2d: its weight, bias, stride and padding; output_padding 0) of a pixel-major
    activation x [N*H*W, Cin(_p)], BEFORE its input activation `in_act`.  Output sizes follow nn.ConvTranspose2d.
    Returns (y [N*Ho*Wo, round_up(Cout, 8)], Geom(N, Ho, Wo)) with the conventions of `conv_strided`."""
    taps, stride = _strided_spec(conv)
    out_geom = strided_geom(conv, geom)
    if in_act != L.ACT_NONE and in_act not in L.DACT_FROM_OUT:
        raise NotImplementedError(f"conv_transposed: input activation {in_act} has no derivative from its output")
    x, xa = _operand(x, in_act)
    y = _TransposedConv.apply(x, xa.detach() if xa is not x else xa, conv.weight, conv.bias, tuple(geom),
                              tuple(out_geom), taps, stride, in_act, emit, out_f32)
    return y, out_geom
