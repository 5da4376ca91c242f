"""The pixel-major stages of VAE / BetaVAE, VQ-VAE and VQ-VAE-2 (models/vae.py, models/vq_vae.py, models/vq_vae_2.py on
nn/pm.py and nn/vq.py): a stage table, float64 references of every stage and element-wise bounds.  Shared by
tests/test_conv_stack_bounds_cpu.py and tests/test_conv_stack_stages_gpu.py; not a test module.

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
magnitude.  An output stored in bf16 adds U8 of itself; ReLU is 1-Lipschitz, so an activated output inherits its
input's bound.  A gradient the reference passes through unchanged is bit-exact: dres (in the residual's dtype) and
every pad column of every output and gradient, which must be +0.0."""

import collections

import torch
from torch.nn import functional as F

import _vae_reference as V
import _vq_vae_reference as VQ

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U24, U8 = 2.0 ** -24, 2.0 ** -8
RELU, NONE = "relu", None

Layer = collections.namedtuple("Layer", "kind stride pad in_act act res")


# ----------------------------------------------------------------------------------------------------------------------
# stage table
# ----------------------------------------------------------------------------------------------------------------------
def _res_stack(T, key, n_blocks, post_act):
    for b in range(n_blocks):
        k = f"{key}._net.{b}._net"
        T[f"{k}.1"] = Layer("conv", 1, 1, NONE if (post_act and b == 0) else RELU, "next", None)
        T[f"{k}.3"] = Layer("conv", 1, 0, RELU, None, f"{k}.1")


def _encoder(T, state, key):
    k = V._n_strided(state, key + ".")
    for j in range(k):
        T[f"{key}.{2 * j}"] = Layer("strided", 2, 1, NONE, "own", None)
    _res_stack(T, f"{key}.{2 * k}", VQ._n_blocks(state, f"{key}.{2 * k}"), k > 0)
    T[f"{key}.{2 * k + 1}"] = Layer("conv", 1, 1, RELU, None, None)


def _decoder(T, state, key):
    T[f"{key}.0"] = Layer("conv", 1, 1, NONE, None, None)
    _res_stack(T, f"{key}.1", VQ._n_blocks(state, f"{key}.1"), False)
    k = V._n_strided(state, key + ".")
    j = 2
    for t in range(k):
        T[f"{key}.{j}"] = Layer("transposed", 2, 1, RELU if t == 0 else NONE, "own" if t < k - 1 else None, None)
        j += 2 if t < k - 1 else 1


def table(state):
    """{parameter prefix: Layer} of a VAE, VQ-VAE or VQ-VAE-2 state dict, in the reference's forward order."""
    T = {}
    tops = sorted({k.split(".")[0] for k in state})
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
        ratio = torch.where(exact, (err > 0).to(F64) * float("inf"), err / bound.clamp_min(1e-300))
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


def _relu_out(a):
    return (a.to(F64) > 0).to(F64)


def _linear(layer, x, w):
    if layer.kind == "transposed":
        return F.conv_transpose2d(x, w, None, stride=layer.stride, padding=layer.pad)
    return F.conv2d(x, w, None, stride=layer.stride, padding=layer.pad)


def stage_in(layer, x):
    """What the stage's contraction reads: its input activation applied to x."""
    return torch.relu(x) if layer.in_act == RELU else x


def stage_y(layer, xa, w, b, res=None):
    """The stage's output before any activation: the contraction of xa, the bias and the residual."""
    y = _linear(layer, xa, w) + b[None, :, None, None]
    return y if res is None else y + res


def stage_out(layer, y):
    """What the next stage receives: ReLU(y) when the stage owns the activation on its output, else y (a `next`
    activation is the consumer's in_act)."""
    return torch.relu(y) if layer.act == "own" else y


def _bf16_store(ref, err):
    """Bound of a bf16 store of a value within err of ref."""
    return err * (1 + U8) + U8 * ref.abs()


def conv_stage(C, name, layer, rec, res_in, weight, bias):
    """Holds one recorded convolution to its float64 reference.  rec: the Recorder's record (args, out, grads, res);
    res_in: the recorded input of the table's residual source (or None)."""
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

    # the operand: bf16(in_act(x)), bit for bit
    xa_ref = (torch.relu(x.float()) if layer.in_act == RELU else x.float()).to(BF16)
    C.equal(f"{label}.xa", xa_got[:, :cin], xa_ref[:, :cin])
    C.zero(f"{label}.xa_pad", xa_got[:, cin:])
    xa64 = nchw(xa_ref, in_geom, cin).clone().requires_grad_(True)
    wv = w64.clone().requires_grad_(True)
    r64 = None if res_in is None else nchw(res_in, out_geom, cout)
    y64 = stage_y(layer, xa64, wv, b64, r64)
    mag = stage_y(layer, xa64.detach().abs(), w64.abs(), b64.abs(), None if r64 is None else r64.abs())
    k_fwd = cin * (T if layer.kind != "transposed" else 1) + (T if layer.kind == "transposed" else 0)
    y, err = pm(y64.detach()), pm((k_fwd + 3) * U24 * mag)

    main, ya = rec.y, rec.ya
    if main is not None:
        if main.dtype == F32:
            C.within(f"{label}.y", main[:, :cout], y, err)
        else:
            C.within(f"{label}.y", main[:, :cout], y, _bf16_store(y, err))
        C.zero(f"{label}.y_pad", main[:, cout:])
    if ya is not None:
        act = torch.relu(y) if layer.act else y  # an own ReLU, or the consumer's (`next`) on the operand it emits
        C.within(f"{label}.ya", ya[:, :cout], act, _bf16_store(act, err))
        C.zero(f"{label}.ya_pad", ya[:, cout:])

    # backward: the gradient w.r.t. y, as the bf16 GEMM operand
    if rec.grads is None:
        return
    g = None
    for gi, wrt in zip(rec.grads, (main, ya)):
        if gi is None:
            continue
        gi = gi[:, :cout].to(F64)
        if wrt is ya and layer.act == "own":  # the stage's own ReLU, from its activated output
            gi = gi * _relu_out(ya[:, :cout])
        g = gi if g is None else g + gi
    if g is None:
        return
    gb = g.to(F32).to(BF16).to(F64)
    gb4 = nchw(gb, out_geom, cout)
    dxa, dw = torch.autograd.grad(y64, (xa64, wv), gb4, retain_graph=True)
    xa_abs = xa64.detach().abs().requires_grad_(True)
    w_abs = w64.abs().requires_grad_(True)
    mag_x, mag_w = torch.autograd.grad(_linear(layer, xa_abs, w_abs), (xa_abs, w_abs), gb4.abs())
    P_out, P_in = gb.shape[0], xa_ref.shape[0]
    dx_g, dw_g, db_g, dres_g = rec.dx, rec.dw, rec.db, rec.dres

    if dw_g is not None:
        k_w = (P_out if layer.kind != "transposed" else P_in) + 64 + 132 + 3
        C.within(f"{label}.dw", dw_g, dw, k_w * U24 * mag_w)
    if db_g is not None:
        C.within(f"{label}.db", db_g, gb.sum(0), (P_out + 64 + 132 + 3) * U24 * gb.abs().sum(0))
    if dx_g is not None:
        d = pm(dxa)
        m = pm(mag_x)
        if layer.in_act == RELU:
            mask = _relu_out(xa_ref[:, :cin])
            d, m = d * mask, m * mask
        k_x = cout * T + T + 3
        err = k_x * U24 * m
        if rec.bf16_partials:
            err = err + U8 * m
        if dx_g.dtype == BF16:
            err = _bf16_store(d, err)
        C.within(f"{label}.dx", dx_g[:, :cin], d, err)
        C.zero(f"{label}.dx_pad", dx_g[:, cin:])
    if rec.has_res:
        # d res = dy: the incoming gradient itself, in the residual's dtype
        C.equal(f"{label}.dres", dres_g if dres_g is not None else torch.empty(0), g.to(rec.res_dtype))


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
