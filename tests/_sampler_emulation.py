"""fp32 CPU stand-ins for the `_lib` entry points the incremental sampler's per-pixel programs reach
(models/incremental.py and the `_pixel_program` of PixelCNN, GatedPixelCNN, PixelSNAIL and ImageGPT), so that the
product's own `IncrementalSamplingMixin.sample` runs without a GPU.  The GEMM, activations, gates, LayerNorm and the
window convolution are tests/_conv_stack_emulation.py's and tests/_block_emulation.py's; the KV-cached attention step
is new here.  Shared by tests/test_sampler_bounds_cpu.py; not a test module.

`attn_decode` follows pg_attn_decode's rounding points: it writes the new key / value row at `pos` before it reads
rows <= pos (< pos when strict), sums scores, the softmax and P V in fp32 with P kept in fp32, and rounds o to bf16
once; a strict row 0 has no key and gets o = 0."""

import ctypes
import math

import numpy as np
import torch

import _block_emulation as BE
import _conv_stack_emulation as CE

F32, BF16 = torch.float32, torch.bfloat16


def gemm(*a, act=0, **kw):
    """The conv-stack GEMM for ReLU / ELU epilogues, the fused block's for GELU (act 2)."""
    return (BE.gemm if act & 0xFF == BE.ACT_GELU else CE.gemm)(*a, act=act, **kw)


def attn_decode(q, k_new, v_new, k_cache, v_cache, o, pos_dev, N, S, H, dk, dv, strict, dk_true=None):
    p = int(pos_dev.reshape(-1)[0])
    kc, vc = k_cache.view(N, S, -1), v_cache.view(N, S, -1)
    kc[:, p, : H * dk] = k_new[:, : H * dk]  # the new row first: a non-strict step attends to it
    vc[:, p, : H * dv] = v_new[:, : H * dv]
    nkeys = p if strict else p + 1
    scale = 1.0 / math.sqrt(dk_true or dk)
    for h in range(H):
        if nkeys == 0:
            o[:, h * dv: (h + 1) * dv] = 0
            continue
        qh = q[:, h * dk: (h + 1) * dk].float()
        kh = kc[:, :nkeys, h * dk: (h + 1) * dk].float()
        vh = vc[:, :nkeys, h * dv: (h + 1) * dv].float()
        s = torch.einsum("nd,nsd->ns", qh, kh) * scale
        e = torch.exp(s - s.amax(1, keepdim=True))
        o[:, h * dv: (h + 1) * dv] = (torch.einsum("ns,nsd->nd", e, vh) / e.sum(1, keepdim=True)).to(BF16)


def cast_multi(src_ptrs, dst_ptrs, numel, chunks, n_chunks, chunk_elems):
    """fp32 -> bf16 of every (source, destination) pointer pair: ImageGPT's packing of weights whose heads fill their
    slots.  CPU memory, read and written through the addresses the kernel would get."""
    for s, d, k in zip(src_ptrs.tolist(), dst_ptrs.tolist(), numel.tolist()):
        src = np.ctypeslib.as_array((ctypes.c_float * k).from_address(s))
        dst = np.ctypeslib.as_array((ctypes.c_int16 * k).from_address(d))
        dst[:] = torch.from_numpy(src.copy()).to(BF16).view(torch.int16).numpy()


STAND_INS = dict(CE.STAND_INS, gemm=gemm, layernorm_fwd=BE.layernorm_fwd, attn_decode=attn_decode,
                 cast_multi=cast_multi)


class _CudaLike:
    """What `_incremental_ok` reads of a canvas, as if it lived on the GPU."""

    def __init__(self, canvas):
        self.shape, self.is_cuda = canvas.shape, True


class _NoCapture:
    def __init__(self, *a, **kw):
        raise RuntimeError("CUDA-graph capture is not available on the CPU")


def install(monkeypatch):
    """Replaces the `_lib` entry points with the stand-ins, and lets the sampler run its eager path on CPU tensors:
    `_incremental_ok` sees a CUDA-like canvas (every other condition it checks still holds), `torch.cuda.synchronize`
    does nothing and the graph capture fails, so `sample()` launches the program eagerly."""
    from pytorch_generative_b200 import _lib
    from pytorch_generative_b200.models import gated_pixel_cnn, image_gpt, incremental, pixel_snail

    for name, fn in STAND_INS.items():
        monkeypatch.setattr(_lib, name, fn)
    for cls in (incremental.IncrementalSamplingMixin, gated_pixel_cnn.GatedPixelCNN, pixel_snail.PixelSNAIL,
                image_gpt.ImageGPT):
        ok = cls.__dict__["_incremental_ok"]
        monkeypatch.setattr(cls, "_incremental_ok", lambda self, canvas, ok=ok: ok(self, _CudaLike(canvas)))
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **kw: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _NoCapture)
