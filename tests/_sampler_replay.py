"""Drives the incremental sampler for the per-pixel stage tests: builds a model with parameters away from their initial
values, records every primitive of its per-pixel program while `IncrementalSamplingMixin.sample` runs it eagerly,
holds each record to its stage of tests/_sampler_reference.py and every hand-off to the stage graph, and keeps the bug
models the replay must reject.  Shared by tests/test_sampler_bounds_cpu.py and tests/test_sampler_stages_gpu.py; not
a test module.

Checks (names '<kind> <stage>@<pixel>.<what>', grouped by `_conv_stack_reference.kind_of`):
  * stage values: every recorded output within its bound of the float64 reference of its recorded inputs;
  * hand-offs, bit for bit (`handoff`): every operand and residual equals what the graph names — the value an earlier
    stage of the step recorded, or cache rows, each the value its writing stage recorded at its write step or zero
    padding, or the final canvas (so an image value that was not final when it went in fails).  The fix-ups of pixel 0
    redo row 0, which pixel 1 finishes: their operands are not final and only their values are checked;
  * `rows`: at step p the program writes row p of each cache, plus row p - 1 of the fix-up caches, and nothing else;
  * `cache`: after the run, every cache row holds its writer's recorded value (rows no step finishes excepted) and the
    zero row is zero;
  * `logits`: what `sample_fn` receives is the last stage's output, unpermuted;
  * `pad`: every pad column of every operand, output and cache row is +0.0."""

import types

import torch

import _conv_stack_reference as CR
import _sampler_reference as R
from _conv_stack_replay import _mutate_fn

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16

CLASSES = {"pixel_cnn": "PixelCNN", "gated_pixel_cnn": "GatedPixelCNN", "pixel_snail": "PixelSNAIL",
           "image_gpt": "ImageGPT"}


def build(model, kwargs, seed=0, device="cpu"):
    """A model of `kwargs` whose biases (and ImageGPT's positional encoding) are N(0, 0.5^2)."""
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = getattr(models, CLASSES[model])(**kwargs)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("bias") or name == "_pos":
                p.copy_(0.5 * torch.randn(p.shape, generator=g))
    return m.to(device)


def start_canvas(shape, conditioned, seed, device):
    """-1 everywhere (unconditional), or with the top rows and the first pixels of the next row given (values on the
    model's grid)."""
    n, c, h, w = shape
    canvas = torch.full(shape, -1.0)
    if conditioned:
        g = torch.Generator().manual_seed(seed + 7)
        r = max(h // 3, 1)
        canvas[:, :, :r] = (torch.rand(n, c, r, w, generator=g) < 0.5).float()
        canvas[:, :, r, : w // 2] = (torch.rand(n, c, w // 2, generator=g) < 0.5).float()
    return canvas.to(device)


class UniformSampleFn:
    """A deterministic `sample_fn` from pre-drawn uniforms (one [n, C] per pixel, in raster order): a Bernoulli draw of
    sigmoid(logits) for C logits, an inverse-CDF draw of each channel's class for K C logits (class k of channel c at
    k C + c) returning k / (K - 1).  It keeps a copy of every logits tensor it is handed."""

    def __init__(self, uniforms, classes=None):
        self.u, self.classes, self.i, self.seen = uniforms, classes, 0, []

    def __call__(self, logits):
        self.seen.append(logits.clone())
        u = self.u[self.i].to(logits.device)
        self.i += 1
        if self.classes is None:
            return (u < torch.sigmoid(logits.float())).float()
        n = logits.shape[0]
        p = torch.softmax(logits.double().reshape(n, self.classes, -1), 1).cumsum(1)
        k = (p < u.double().unsqueeze(1)).sum(1).clamp_max(self.classes - 1)
        return k.float() / (self.classes - 1)


def uniforms(shape, seed):
    n, c, h, w = shape
    g = torch.Generator().manual_seed(seed + 11)
    return [torch.rand(n, c, generator=g) for _ in range(h * w)]


# ----------------------------------------------------------------------------------------------------------------------
# the recorder
# ----------------------------------------------------------------------------------------------------------------------
def row_caches(model, st, n, S):
    """{graph cache name: the product's cache as [n, rows, width]}."""
    out = {}
    if model != "image_gpt":
        out["image"] = st["image"]
    if model == "pixel_cnn":
        out.update({f"t1.{i}": t for i, t in enumerate(st["t1"])})
    elif model == "gated_pixel_cnn":
        out.update({f"vc.{i}": t for i, t in enumerate(st["vc"])})
        out.update({f"hc.{i}": t for i, t in enumerate(st["hc"])})
    elif model == "pixel_snail":
        for bi, b in enumerate(st["blocks"]):
            out.update({f"ea.{bi}.{j}": t for j, t in enumerate(b["ea"])})
            out.update({f"eb.{bi}.{j}": t for j, t in enumerate(b["eb"])})
            out[f"kc.{bi}"], out[f"vc.{bi}"] = b["kc"].view(n, S, -1), b["vc"].view(n, S, -1)
    else:
        for b in range(len(st["kc"])):
            out[f"kc.{b}"], out[f"vc.{b}"] = st["kc"][b].view(n, S, -1), st["vc"][b].view(n, S, -1)
    return out


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


class Recorder:
    """Wraps the program's primitives (ops.linear_fwd, _lib.act_cast, pm.gated, pm.gated_res, _lib.attn_decode,
    ops.layernorm_fwd, _lib.conv_small_fwd) and the model's `_start_pixels`, `_before_pixel`, `_after_pixel` and
    `sample_fn`.  Records are kept per pixel from the first `_start_pixels` on (the warm-up launch before it is not a
    pixel).  After each pixel it notes which rows of each cache changed (from snapshots: the fix-ups write with
    index_copy_, which no wrapper sees).  `snap`: the pixels whose decode records keep the K / V rows they read (None:
    every pixel)."""

    def __init__(self, monkeypatch, m, model, snap=None):
        from pytorch_generative_b200 import _lib, ops
        from pytorch_generative_b200.nn import pm

        self.model, self.snap = model, snap
        self.steps, self.changed, self.logits = [], [], []
        self.active, self.st = False, None
        rec = self

        def add(**kw):
            if rec.active:
                rec.steps[-1].append(types.SimpleNamespace(**kw))

        linear_fwd, layernorm_fwd = ops.linear_fwd, ops.layernorm_fwd
        act_cast, attn_decode, conv_small_fwd = _lib.act_cast, _lib.attn_decode, _lib.conv_small_fwd
        gated, gated_res = pm.gated, pm.gated_res

        def linear(a, w, bias=None, *, act=0, res0=None, res1=None, **kw):
            out = linear_fwd(a, w, bias, act=act, res0=res0, res1=res1, **kw)
            add(kind="linear", a=a.clone(), res=[r.clone() for r in (res0, res1) if r is not None], act=act,
                b=out[0], f=out[2])
            return out

        def act(x, a, out):
            act_cast(x, a, out)
            add(kind="act", x=x.clone(), act=a, out=out.clone())

        def gate(x, a, dtype=BF16):
            y = gated(x, a, dtype)
            add(kind="gate", x=x.clone(), out=y)
            return y

        def gres(x, res, a):
            y = gated_res(x, res, a)
            add(kind="gated_res", x=x.clone(), res=res.clone(), out=y)
            return y

        def decode(q, k, v, kc, vc, o, pos, N, S, H, dk, dv, strict, dk_true=None):
            attn_decode(q, k, v, kc, vc, o, pos, N, S, H, dk, dv, strict, dk_true=dk_true)
            p = len(rec.steps) - 1
            keep = rec.active and (rec.snap is None or p in rec.snap)
            add(kind="decode", q=q.clone(), k=k.clone(), v=v.clone(), o=o.clone(), strict=strict,
                kc=kc.view(N, S, -1)[:, : p + 1].clone() if keep else None,
                vc=vc.view(N, S, -1)[:, : p + 1].clone() if keep else None)

        def ln(x, gamma, beta, eps, *a, **kw):
            out = layernorm_fwd(x, gamma, beta, eps, *a, **kw)
            add(kind="ln", x=x.clone(), out=out[0])
            return out

        def conv_small(x, w, b, pad, out_f32=None, **kw):
            conv_small_fwd(x, w, b, pad, out_f32=out_f32, **kw)
            add(kind="conv_small", x=x.clone(), out=out_f32.clone())

        for owner, name, fn in ((ops, "linear_fwd", linear), (ops, "layernorm_fwd", ln), (_lib, "act_cast", act),
                                (_lib, "attn_decode", decode), (_lib, "conv_small_fwd", conv_small),
                                (pm, "gated", gate), (pm, "gated_res", gres)):
            monkeypatch.setattr(owner, name, fn)

        cls = type(m)

        def start(st, canvas):
            cls._start_pixels(m, st, canvas)
            rec.st, rec.active = st, True
            rec.n, rec.S = canvas.shape[0], canvas.shape[2] * canvas.shape[3]
            rec.snaps = {k: v.clone() for k, v in row_caches(model, st, rec.n, rec.S).items()}

        def before(sp, st, canvas, row, col):
            rec.steps.append([])
            cls._before_pixel(m, sp, st, canvas, row, col)

        def after(sp, st, new, row, col):
            cls._after_pixel(m, sp, st, new, row, col)
            rows = {}
            for k, t in row_caches(model, st, rec.n, rec.S).items():
                d = (_bits(t) != _bits(rec.snaps[k])).flatten(2).any(2).any(0)
                rows[k] = set(d.nonzero().flatten().tolist())
                rec.snaps[k] = t.clone()
            rec.changed.append(rows)

        fn = m._sample_fn

        def sample_fn(logits):
            rec.logits.append(logits.clone())
            return fn(logits)

        m.__dict__.update(_start_pixels=start, _before_pixel=before, _after_pixel=after, _sample_fn=sample_fn)


# ----------------------------------------------------------------------------------------------------------------------
# the replay
# ----------------------------------------------------------------------------------------------------------------------
def _t(x, cols):
    return x.detach()[:, cols].to(F64).cpu()


def _pads(C, label, x, lay):
    cols = R.pad_cols(lay)
    if cols:
        C.zero(label, x.detach()[..., cols].cpu())


def _same(C, label, got, ref):
    """Bit for bit (as float64 values of the same bf16 / fp32 numbers)."""
    C.within(label, got, ref.to(got.device), torch.zeros_like(ref, dtype=F64))


def replay(G, rec, canvas, pixels=None):
    """Every check of the module docstring; pixels: the pixels whose stages and hand-offs are checked (None: all).
    Returns the Checks."""
    C = CR.Checks()
    env = R.Env(G, canvas.detach().cpu(), exact=False)
    stages = G.recorded()
    for p in range(G.S):
        recs = rec.steps[p]
        want = [s.kind for s in stages]
        got = [r.kind for r in recs]
        if got != want:
            C.failures[f"program @{p}.stages"] = f"pixel {p}: recorded {got}, the graph has {want}"
            return C
        it = iter(recs)
        check = pixels is None or p in pixels
        for st in G.stages:
            if st.kind == "virtual":
                env.vals[p][st.name] = {"f": env.ev(st.src, p)}
                continue
            r = next(it)
            env.vals[p][st.name] = _stage(C, env, st, r, p, check, handoffs=check and not (p == 0 and
                                                                                      getattr(st, "fixup", False)))
        if check:
            _same(C, f"logits @{p}.order", rec.logits[p].to(F64).cpu(), recs[-1].f.to(F64).cpu())
            if rec.logits[p].shape != recs[-1].f.shape:
                C.failures[f"logits @{p}.order"] = f"pixel {p}: logits of shape {tuple(rec.logits[p].shape)}"
            for name, rows in rec.changed[p].items():
                allowed = {p} | ({max(p - 1, 0)} if G.caches[name].lag else set())
                if rows - allowed:
                    C.failures[f"rows {name}@{p}.written"] = f"pixel {p} wrote rows {sorted(rows - allowed)} of {name}"
                else:
                    C.ratios[f"rows {name}@{p}.written"] = 0.0
    caches = row_caches(G.model, rec.st, G.n, G.S)
    for name, t in caches.items():
        spec = G.caches[name]
        rows = [r for r in range(G.S) if r + spec.lag < G.S]
        got = t[:, rows].detach().cpu()
        ref = torch.stack([env.cache_row(name, r) for r in rows], 1)
        _same(C, f"cache {name}.final", got[..., spec.layout.cols].to(F64), ref)
        _pads(C, f"pad {name}.cache", got, spec.layout)
        if t.shape[1] > G.S:  # the zero row of the taps outside the image
            C.zero(f"cache {name}.zero_row", t[:, G.S:].detach().cpu())
    return C


def _stage(C, env, st, r, p, check, handoffs):
    """Checks one record against its stage; returns the stage's values (true channels, float64, CPU)."""
    lbl = lambda kind, what: f"{kind} {st.name}@{p}.{what}"
    lo = st.lay_out
    if st.kind == "linear":
        vals = {}
        if r.f is not None:
            vals["f"] = _t(r.f, lo.cols)
        if r.b is not None:
            vals["b"] = _t(r.b, lo.cols)
        if not check:
            return vals
        a = _t(r.a, st.lay_in.cols)
        res = [_t(x, lo.cols) for x in r.res]
        if handoffs:
            _same(C, lbl("handoff", "a"), a, env.ev(st.src, p))
            if len(res) != len(st.res):
                C.failures[lbl("handoff", "res")] = f"{st.name} @ {p}: {len(res)} residuals, the graph has {len(st.res)}"
            for i, (x, spec) in enumerate(zip(res, st.res)):
                _same(C, lbl("handoff", f"res{i}"), x, env.ev(spec, p))
        if st.pads:
            _pads(C, lbl("pad", "a"), r.a, st.lay_in)
        y, mag = R.linear_ref(st, a, res)
        bounds = R.linear_bound(st, r.a.shape[1], y, mag)
        for which in ("f", "b"):
            if which in vals:
                ref, err = bounds[which]
                C.within(lbl("linear", "y" if which == "f" else "yb"), vals[which], ref, err)
                _pads(C, lbl("pad", "y" + which), getattr(r, which), lo)
        return vals
    if st.kind == "act":
        out = _t(r.out, lo.cols)
        if check:
            x = _t(r.x, st.lay_in.cols)
            if handoffs:
                _same(C, lbl("handoff", "a"), x, env.ev(st.src, p))
            if r.act != st.act:
                C.failures[lbl("act", "kind")] = f"{st.name} @ {p}: activation {r.act}, the graph has {st.act}"
            ref, err, exact = R.act_ref(st, x)
            C.within(lbl("act", "y"), out, ref, torch.zeros_like(ref) if exact else err)
            _pads(C, lbl("pad", "y"), r.out, lo)
        return {"b": out}
    if st.kind in ("gate", "gated_res"):
        out = _t(r.out, lo.cols)
        if check:
            x = _t(r.x, st.lay_in.cols)
            if handoffs:
                _same(C, lbl("handoff", "a"), x, env.ev(st.src, p))
            Cc = x.shape[1] // 2
            act = R.TANH if st.kind == "gate" else R.NONE
            y, err = R.gate_refb(x, r.x.dtype, Cc, act)
            if st.kind == "gate":
                C.within(lbl("gate", "y"), out, y, err * (1 + R.U8) + R.U8 * y.abs())
            else:
                res = _t(r.res, lo.cols)
                if handoffs:
                    _same(C, lbl("handoff", "res0"), res, env.ev(st.res[0], p))
                y = y + res
                C.within(lbl("gated_res", "y"), out, y, err + R.U24 * (y.abs() + err))
            _pads(C, lbl("pad", "y"), r.out, lo)
        return {"f" if st.f32 else "b": out}
    if st.kind == "ln":
        out = _t(r.out, lo.cols)
        if check:
            x = _t(r.x, st.lay_in.cols)
            if handoffs:
                _same(C, lbl("handoff", "a"), x, env.ev(st.src, p))
            y, err = R.ln_ref(st, x)
            C.within(lbl("ln", "y"), out, y, err)
            _pads(C, lbl("pad", "y"), r.out, lo)
        return {"b": out}
    if st.kind == "conv_small":
        out = _t(r.out, lo.cols)
        if check:
            x = r.x.detach().to(F64).cpu()
            if handoffs:
                live = st.mask.bool()
                _same(C, lbl("handoff", "patch"), x[:, :, live], env.patch(p)[:, :, live])
            y, err = R.conv_small_ref(st, x)
            C.within(lbl("conv_small", "y"), out, y, err)
            _pads(C, lbl("pad", "y"), r.out, lo)
        return {"f": out}
    assert st.kind == "decode", st.kind
    out = _t(r.o, lo.cols)
    if check:
        kcols = R.slots(st.H, st.dk, st.qs).cols
        vcols = R.slots(st.H, st.dv, st.vs).cols
        q, k, v = _t(r.q, kcols), _t(r.k, kcols), _t(r.v, vcols)
        if handoffs:
            eq, ek, ev_ = R._qkv(env, st, p, env.ev(st.src, p))
            for what, got, ref in (("q", q, eq), ("k", k, ek), ("v", v, ev_)):
                _same(C, lbl("handoff", what), got, ref)
        if r.strict != st.strict:
            C.failures[lbl("decode", "strict")] = f"{st.name} @ {p}: strict={r.strict}, the graph has {st.strict}"
        if r.kc is not None:
            kc, vc = r.kc.detach().cpu(), r.vc.detach().cpu()
            kt, vt = kc[..., kcols].to(F64), vc[..., vcols].to(F64)
            if handoffs and p > 0:  # the rows it read: each the value its writer recorded at its write step
                _same(C, lbl("handoff", "kc"), kt[:, :p], torch.stack([env.cache_row(st.kc, j) for j in range(p)], 1))
                _same(C, lbl("handoff", "vc"), vt[:, :p], torch.stack([env.cache_row(st.vc, j) for j in range(p)], 1))
            _same(C, lbl("decode", "k_row"), kt[:, p], k)
            _same(C, lbl("decode", "v_row"), vt[:, p], v)
            _pads(C, lbl("pad", "kc"), kc, R.slots(st.H, st.dk, st.qs))
            ref, err = R.decode_ref(st, q, kt, vt, p, st.strict)
            C.within(lbl("decode", "o"), out, ref, err)
        _pads(C, lbl("pad", "o"), r.o, lo)
    return {"b": out}


def run(m, model, kwargs, shape, conditioned, monkeypatch, seed=0, snap=None, classes=None, graph_mode=False):
    """One recorded sample() of m: (Graph, Recorder, final canvas).  graph_mode: leave the capture alone (the GPU's
    captured run, unrecorded); otherwise the capture is made to fail and the program runs eagerly."""
    m._sample_fn = UniformSampleFn(uniforms(shape, seed), classes)
    canvas = start_canvas(shape, conditioned, seed, next(m.parameters()).device)
    rec = Recorder(monkeypatch, m, model, snap)
    out = m.sample(conditioned_on=canvas)
    state = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    G = R.graph(model, state, tuple(shape), kwargs.get("n_attention_heads"))
    return G, rec, out


# ----------------------------------------------------------------------------------------------------------------------
# bug models: each changes one thing the product does
# ----------------------------------------------------------------------------------------------------------------------
def _inc():
    from pytorch_generative_b200.models import incremental
    return incremental


def bug_taps_wrap_rows(monkeypatch):
    """The tap table checks the flat index only, not the column: a tap left of column 0 reads the last pixel of the
    row above it instead of the zero row."""
    _mutate_fn(monkeypatch, _inc().PixelStepper, "table", "ok = (r >= 0) & (r < self.h) & (c >= 0) & (c < self.w)",
               "ok = (r * self.w + c >= 0) & (r * self.w + c < self.S)")


def bug_valid_mask_off_by_one(monkeypatch):
    from pytorch_generative_b200.models import gated_pixel_cnn
    _mutate_fn(monkeypatch, gated_pixel_cnn.GatedPixelCNN, "_build_pixel_state", "- layer._padding - 1) >= 0",
               "- layer._padding) >= 0")


def bug_vstack_fixup_reads_pos(monkeypatch):
    from pytorch_generative_b200.models import gated_pixel_cnn
    _mutate_fn(monkeypatch, gated_pixel_cnn.GatedPixelCNN, "_pixel_program",
               'vin = st["image"].index_select(1, sp.prev)[:, 0]', 'vin = st["image"].index_select(1, sp.pos)[:, 0]')


def bug_kv_fixup_skipped(monkeypatch):
    """PixelSNAIL recomputes row p - 1's key / value from the operand it still holds: the placeholder image value."""
    from pytorch_generative_b200.models import pixel_snail
    _mutate_fn(monkeypatch, pixel_snail.PixelSNAIL, "_pixel_program", 'b["akv"][:, 2 + C: 2 + C + c] = prev_img',
               "pass")


def bug_decode_not_strict(monkeypatch):
    from pytorch_generative_b200.models import pixel_snail
    _mutate_fn(monkeypatch, pixel_snail.PixelSNAIL, "_pixel_program", "True, dk_true=blk._attention._embed_channels)",
               "False, dk_true=blk._attention._embed_channels)")


def bug_xin_without_pos(monkeypatch):
    from pytorch_generative_b200.models import image_gpt
    _mutate_fn(monkeypatch, image_gpt.ImageGPT, "_after_pixel", "= new + self._pos[0, :, row, col]", "= new")


def bug_stream_rounded_to_bf16(monkeypatch):
    from pytorch_generative_b200.models import pixel_cnn
    _mutate_fn(monkeypatch, pixel_cnn.PixelCNN, "_pixel_program", "res0=x, res1=x, f32=True)",
               "res0=x, res1=x, f32=True).to(torch.bfloat16).float()", dict(torch=torch))


def bug_pad_rows_not_zeroed(monkeypatch):
    _mutate_fn(monkeypatch, _inc(), "pad_rows", "wp = torch.zeros(rows, w.shape[1]", "wp = torch.ones(rows, w.shape[1]")


def bug_logits_channel_major(monkeypatch):
    """sample() hands sample_fn the logits in (channel, class) order instead of (class, channel)."""
    _mutate_fn(monkeypatch, _inc().IncrementalSamplingMixin, "sample", "drawn = self._sample_fn(logits)",
               "drawn = self._sample_fn(logits.reshape(n, -1, c).transpose(1, 2).reshape(n, -1))")


# name -> (apply(monkeypatch), the check kind (CR.kind_of) that must fail, the geometry that runs the code it changes)
BUGS = {
    "taps_wrap_rows": (bug_taps_wrap_rows, "handoff.a", "pixel_cnn"),
    "valid_mask_off_by_one": (bug_valid_mask_off_by_one, "handoff.a", "gated"),
    "vstack_fixup_reads_pos": (bug_vstack_fixup_reads_pos, "handoff.a", "gated"),
    "kv_fixup_skipped": (bug_kv_fixup_skipped, "handoff.a", "snail"),
    "decode_not_strict": (bug_decode_not_strict, "decode.o", "snail"),
    "xin_without_pos": (bug_xin_without_pos, "handoff.patch", "gpt"),
    "stream_rounded_to_bf16": (bug_stream_rounded_to_bf16, "handoff.res0", "pixel_cnn"),
    "pad_rows_not_zeroed": (bug_pad_rows_not_zeroed, "pad.yb", "pixel_cnn"),
    "logits_channel_major": (bug_logits_channel_major, "logits.order", "categorical"),
}
