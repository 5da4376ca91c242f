"""Incremental sampling for all four models: one per-pixel program per model, one raster loop.

`AutoregressiveModel.sample` (reference models/base.py:97-120) runs one full forward per pixel.  Every model on the path is
exactly causal, so the logits of pixel p only need, per layer, the activations of the pixels its taps reach — which are
pixels generated earlier.  The convolutional models keep one activation cache `[n, H*W + 1, C]` (bf16, the extra row
stays zero = the convolution's zero padding) per convolution input in a `PixelStepper` and evaluate the stack at ONE
position per image:

    gather   the taps of position p from the layer's cache        (index tables built once, position read on the device)
    linear   [n, taps * C] x W^T on the skinny GEMM (`pg_gemm_bf16` impl 2: weights streamed once, all SMs), with the
             bias / activation / residual epilogues of training; an operand too large for it (more than 160 KiB: a
             wide MLP or tap gather at 32 images) runs on the tensor-core GEMM (`ops.linear_impl`)
    write    the layer's output row into the next layer's cache

Every cache and operand of a convolutional program has `pitch(C) = round_up(C, 8)` columns whose pad columns are
exactly zero, the 16-byte operand pitch of the training stacks, so any channel count samples incrementally.  `pack`
owns that layout on the weight side: zero input columns (`ops.pack_taps`) and zero output rows and bias entries, so
each layer's output already has its pad columns at zero; a gate's input keeps each half at its own pitch
(`parts=2`), so the gate's output is padded the same way (act(0) * sigmoid(0) = 0).  At C % 8 == 0 the layout is the
identity and the operands are those of the unpadded program.

ImageGPT evaluates its input convolution on the window around p and attends over K/V caches (`pg_attn_decode`);
PixelSNAIL combines both.  A model describes its per-pixel program in `_pixel_program(stepper, state)`; the whole
program is captured in one CUDA graph whose position lives in device memory and is replayed H*W times.  The raster
order, the `sample_fn` hook, the "only entries < 0 are overwritten" rule, the weight refresh and the capture are
`IncrementalSamplingMixin.sample`'s.
"""

import warnings

import torch

from .. import _lib as L
from .. import ops

BF16 = torch.bfloat16
MAX_ROWS = ops.SKINNY_ROWS  # images sampled at once by the convolutional programs (their gathers live on the skinny GEMM)


def pitch(channels, parts=1):
    """Columns of a per-pixel cache or operand holding `channels` true channels made of `parts` equal parts (a gate's
    [a | b] input: 2), each part at the 16-byte operand pitch."""
    return parts * ops.round_up(channels // parts, 8)


def _padded_index(channels, parts, device):
    """Column of each true channel in the `pitch(channels, parts)` layout; None where that layout is the identity."""
    part = channels // parts
    step = ops.round_up(part, 8)
    if step == part:
        return None
    return torch.cat([torch.arange(part) + g * step for g in range(parts)]).to(device)


def pad_rows(w, bias, parts=1):
    """A packed GEMM operand `w` [Cout, K] (bf16) and its fp32 bias with their output rows in the padded layout: zero
    rows and bias entries in the pad, so the layer's output columns there are exactly zero.  Returns the inputs
    themselves where the layout is the identity."""
    bias = bias.detach()
    idx = _padded_index(w.shape[0], parts, w.device)
    if idx is None:
        return w, bias
    rows = pitch(w.shape[0], parts)
    wp = torch.zeros(rows, w.shape[1], dtype=w.dtype, device=w.device)
    wp[idx] = w
    bp = torch.zeros(rows, dtype=bias.dtype, device=bias.device)
    bp[idx] = bias
    return wp, bp


def pack(conv, positions=None, *, in_parts=1, out_parts=1):
    """One convolution of a per-pixel program as a GEMM operand: bf16 [pitch(Cout, out_parts), T * pitch(Cin,
    in_parts)], tap-major (`ops.pack_taps`; `positions` as there), and its fp32 bias.  Input columns and output rows
    follow the padded layout, zero in the pad.  out_parts=0: the output keeps its true width (the logits)."""
    cout, cin = conv.weight.shape[:2]
    w = ops.pack_taps(conv.weight, pitch(cin), positions)
    idx = _padded_index(cin, in_parts, w.device) if in_parts > 1 else None
    if idx is not None:  # scatter each tap's columns [0, cin) to the parts' pitches
        taps = w.shape[1] // pitch(cin)
        src = w.view(cout, taps, -1)[:, :, :cin]
        w = torch.zeros(cout, taps, pitch(cin, in_parts), dtype=w.dtype, device=w.device)
        w[:, :, idx] = src
        w = w.view(cout, -1)
    if out_parts == 0:
        return w, conv.bias.detach()
    return pad_rows(w, conv.bias, out_parts)


def live_taps(mask2d, pad_h, pad_w):
    """[(i, j, dy, dx)] of the unmasked kernel positions of a CausalConv2d (row-major, like the weight)."""
    kh, kw = mask2d.shape
    return [(i, j, i - pad_h, j - pad_w) for i in range(kh) for j in range(kw) if float(mask2d[i, j]) != 0.0]


class PixelStepper:
    """Caches, tap tables and the per-pixel primitives for a batch of `n` images of `h x w` pixels."""

    def __init__(self, n, h, w, device):
        self.n, self.h, self.w, self.S, self.device = n, h, w, h * w, device
        self.pos = torch.zeros(1, dtype=torch.int64, device=device)     # current position (device side: graph-replayable)
        self.pos32 = self.pos.view(torch.int32)[:1]  # the same for pg_attn_decode: the low word (0 <= p < 2^31)
        self._tables = {}

    def cache(self, channels):
        """[n, S + 1, pitch(channels)] bf16 zeros: one row per pixel of every image, the pad columns stay zero."""
        return torch.zeros(self.n, self.S + 1, pitch(channels), dtype=BF16, device=self.device)

    def table(self, offsets):
        """[S, T] flat indices of position p's taps (index S = the zero row for taps outside the image)."""
        key = tuple(offsets)
        if key not in self._tables:
            rows = torch.arange(self.h).view(self.h, 1, 1)
            cols = torch.arange(self.w).view(1, self.w, 1)
            dy = torch.tensor([o[0] for o in offsets]).view(1, 1, -1)
            dx = torch.tensor([o[1] for o in offsets]).view(1, 1, -1)
            r, c = rows + dy, cols + dx
            ok = (r >= 0) & (r < self.h) & (c >= 0) & (c < self.w)
            idx = torch.where(ok, r * self.w + c, torch.full_like(r * self.w + c, self.S))
            self._tables[key] = idx.reshape(self.S, len(offsets)).to(self.device)
        return self._tables[key]

    def gather(self, cache, offsets):
        """[n, T * C] bf16: the cache rows under position p's taps, tap-major."""
        idx = self.table(offsets).index_select(0, self.pos)[0]
        return cache.index_select(1, idx).reshape(self.n, -1)

    def write(self, cache, value):
        """cache[:, p, :C] = value ([n, C] of true or padded width; cast to bf16).  The pad columns are left alone."""
        if value.shape[1] != cache.shape[2]:
            cache = cache[:, :, : value.shape[1]]
        cache.index_copy_(1, self.pos, value.to(BF16).unsqueeze(1))

    @staticmethod
    def act(x, act):
        """bf16(act(x)) of an [n, C] row block, any C."""
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
        L.act_cast(x.contiguous(), act, out)
        return out

    @staticmethod
    def linear(a, w, bias, *, act=L.ACT_NONE, res0=None, res1=None, f32=False):
        """a [n, K] bf16 x w [Cout, K]^T (+ bias, residuals) -> bf16(act(.)) or fp32, on the skinny GEMM where it
        takes the operands (`ops.linear_impl`)."""
        ob, _, of = ops.linear_fwd(a, w, bias, act=act, res0=res0, res1=res1, want_bf16=not f32, want_f32=f32, skinny=True)
        return of if f32 else ob


class IncrementalSamplingMixin:
    """`sample()` through a model-specific per-pixel program (`_build_pixel_state`, `_pack_pixel_weights`,
    `_pixel_program`; optionally `_start_pixels`, `_before_pixel`, `_after_pixel`)."""

    _incremental_sampling = True

    def _incremental_ok(self, canvas):
        return self._incremental_sampling and canvas.is_cuda and canvas.shape[0] <= MAX_ROWS

    @torch.no_grad()
    def sample(self, n_samples=None, conditioned_on=None):
        canvas = self._start_canvas(n_samples, conditioned_on)
        if not self._incremental_ok(canvas):
            return super().sample(conditioned_on=canvas)
        n, c, h, w = canvas.shape
        cache = self.__dict__.setdefault("_pixel_states", {})
        key = (n, c, h, w, str(canvas.device))
        st = cache.get(key)
        if st is None:
            st = cache[key] = dict(stepper=PixelStepper(n, h, w, canvas.device), graph=None)
            st.update(self._build_pixel_state(st["stepper"], c))
        self._refresh_pixel_weights(st)          # the weights may have been trained since the last call
        sp = st["stepper"]
        if st["graph"] is None:
            sp.pos.zero_()
            try:
                self._pixel_program(sp, st)      # warm-up outside capture
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    st["logits"] = self._pixel_program(sp, st)
                st["graph"] = graph
            except RuntimeError as exc:
                torch.cuda.synchronize()
                st["graph"], st["graph_error"] = False, repr(exc)
                warnings.warn(f"{type(self).__name__}.sample(): CUDA-graph capture of the per-pixel program failed, "
                              f"launching it eagerly: {exc!r}", RuntimeWarning)
        self._start_pixels(st, canvas)
        for row in range(h):
            for col in range(w):
                sp.pos.fill_(row * w + col)
                self._before_pixel(sp, st, canvas, row, col)
                if st["graph"]:
                    st["graph"].replay()
                    logits = st["logits"]
                else:
                    logits = self._pixel_program(sp, st)
                drawn = self._sample_fn(logits).view(n, c)   # all out_channels logits of the pixel, like base.sample
                current = canvas[:, :, row, col]
                new = torch.where(current < 0, drawn, current)
                canvas[:, :, row, col] = new
                self._after_pixel(sp, st, new, row, col)
        return canvas

    def _start_pixels(self, st, canvas):
        """Hook: reset the state a call must not inherit from the previous one (by default: zero the caches)."""
        for buf in st["caches"]:
            buf.zero_()

    def _before_pixel(self, sp, st, canvas, row, col):
        """Hook: work that must see the previous pixel's final value (PixelSNAIL's key / value fix-up)."""

    def _after_pixel(self, sp, st, new, row, col):
        """Hook: record the pixel just drawn (by default: into the bf16 image cache `st["image"]`)."""
        st["image"][:, row * sp.w + col, : new.shape[1]] = new.to(BF16)

    def _refresh_pixel_weights(self, st):
        for k, v in self._pack_pixel_weights().items():
            if k in st["weights"]:
                st["weights"][k].copy_(v)   # in place: a captured graph keeps reading the same buffers
            else:
                st["weights"][k] = v.clone()  # the sampler's own buffers, never views of a model's other copies
