"""Tap lists of convolutions of any kernel size and dilation, without a GPU: the offsets `conv_taps` builds (row-major,
like the OIHW weight) and that a tap sum over them is nn.Conv2d's dilated convolution cropped to the input; the padding
rule; the choice between the TMA tap loop and the gather path when an offset exceeds 64; the 225-tap limit in Python
and in the C entry points (argument checks that return before any device work); and the CausalConv2d arguments that
stay off the path."""

import ctypes

import pytest
import torch
import torch.nn.functional as F


def test_conv_taps_with_dilation_are_row_major():
    from pytorch_generative_b200.nn.tapconv import conv_taps

    assert conv_taps(3, 3, 1, 1) == tuple((i - 1, j - 1) for i in range(3) for j in range(3))
    assert conv_taps(2, 3, 2, 2, 2, 2) == ((-2, -2), (-2, 0), (-2, 2), (0, -2), (0, 0), (0, 2))
    taps = conv_taps(15, 15, 21, 14, 3, 2)
    assert len(taps) == 225
    assert taps[0] == (-21, -14) and taps[1] == (-21, -12) and taps[15] == (-18, -14) and taps[-1] == (21, 14)


@pytest.mark.parametrize("k,pad,dil", [((3, 3), (1, 1), (1, 1)), ((7, 7), (3, 3), (1, 1)), ((3, 5), (2, 4), (2, 2)),
                                       ((5, 3), (6, 1), (3, 1)), ((2, 2), (1, 1), (1, 1)), ((3, 3), (4, 3), (2, 2))])
def test_tap_sum_is_the_cropped_dilated_conv2d(k, pad, dil):
    """sum_t W_t x[p + off_t] (zero outside the image) over conv_taps == conv2d(x, w, padding, dilation)[:, :, :h, :w],
    the front crop the path computes, in float64."""
    from pytorch_generative_b200.nn.tapconv import conv_taps

    g = torch.Generator().manual_seed(0)
    n, cin, cout, h, w = 2, 3, 4, 9, 11
    x = torch.randn(n, cin, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, cin, *k, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, wt, padding=pad, dilation=dil)[:, :, :h, :w]
    xp = F.pad(x, (64, 64, 64, 64))
    out = torch.zeros(n, cout, h, w, dtype=torch.float64)
    for t, (dy, dx) in enumerate(conv_taps(*k, *pad, *dil)):
        i, j = divmod(t, k[1])
        shifted = xp[:, :, 64 + dy:64 + dy + h, 64 + dx:64 + dx + w]
        out += torch.einsum("oc,nchw->nohw", wt[:, :, i, j], shifted)
    assert torch.allclose(out, ref, rtol=1e-12, atol=1e-12)


def test_padding_rule():
    from pytorch_generative_b200.nn import pm

    w = torch.zeros(8, 8, 7, 5)
    pm._check_padding(w, (3, 2))
    pm._check_padding(w, (6, 4), (2, 2))
    pm._check_padding(w, (9, 2), (3, 1))
    for pad, dil in [((2, 2), (1, 1)), ((3, 2), (2, 1)), ((6, 3), (2, 2)), ((3, 2), (1, 2))]:
        with pytest.raises(NotImplementedError, match="too small"):
            pm._check_padding(w, pad, dil)


def test_tap_loop_takes_offsets_up_to_64_and_gather_the_rest():
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.nn.tapconv import conv_taps

    assert L.MAX_TAP_OFFSET == 64
    assert L.conv_gemm_supported(32, 32, 64)
    assert L.conv_gemm_supported(32, 32, 64, conv_taps(15, 15, 21, 21, 3, 3))
    assert L.conv_gemm_supported(128, 64, 64, conv_taps(3, 3, 64, 64, 64, 64))
    assert not L.conv_gemm_supported(130, 64, 64, conv_taps(3, 3, 65, 1, 65, 1))   # dy = +-65
    assert not L.conv_gemm_supported(130, 64, 64, conv_taps(1, 3, 0, 65, 1, 65))   # dx = +-65
    assert not L.conv_gemm_supported(28, 28, 64, conv_taps(3, 3, 1, 1))            # the image, as before
    assert not L.conv_gemm_supported(32, 32, 100, conv_taps(3, 3, 1, 1))           # the channels, as before


def test_conv_refuses_more_than_225_taps_and_names_the_limit():
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.nn import pm

    assert L.MAX_TAPS == 225
    x = torch.zeros(16, 64, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match=r"226 taps exceed the 225 of the tap kernels \(kernel 2x113"):
        pm.conv(x, torch.zeros(8, 64, 2, 113), None, pm.Geom(1, 4, 4), (1, 56))
    with pytest.raises(NotImplementedError, match=r"256 taps exceed the 225 .*at most 225 kernel positions, e\.g\. 15 x 15"):
        pm.conv(x, torch.zeros(8, 64, 16, 16), None, pm.Geom(1, 4, 4), (8, 8))
    # the limit counts positions, not sides: 1 x 225 and 9 x 25 pass it and reach the CUDA path, which refuses CPU tensors
    for k, pad in [((1, 225), (0, 112)), ((9, 25), (4, 12))]:
        with pytest.raises(RuntimeError, match="CUDA tensors"):
            pm.conv(x, torch.zeros(8, 64, *k), None, pm.Geom(1, 4, 4), pad)


@pytest.fixture(scope="module")
def lib():
    from pytorch_generative_b200 import _build, _lib

    _build.build(verbose=False)
    return _lib.load()


def _error(lib):
    return lib.pg_last_error().decode()


def test_c_entry_points_check_the_tap_limits(lib):
    """The checks return an error before any device work: the pointers below are host buffers never dereferenced."""
    from pytorch_generative_b200 import _lib as L

    buf = torch.zeros(1024, dtype=torch.float32)
    p = buf.data_ptr()
    e = L.GemmEpilogue()
    e.out_f32, e.ld_out_f32 = p, 64

    def taps(vals):
        return ctypes.cast((ctypes.c_int * len(vals))(*vals), ctypes.c_void_p)

    z226 = taps([0] * 226)
    rc = lib.pg_gemm_bf16_conv_taps(p, 64, p, 64, 128, 64, 226 * 64, 1, ctypes.byref(e), L.CONV_FWD, 1, 16, 8, 64, 226,
                                    z226, z226, None)
    assert rc != 0 and "1..225 taps (got 226)" in _error(lib)
    far = taps([0, 65])
    rc = lib.pg_gemm_bf16_conv_taps(p, 64, p, 64, 128, 64, 2 * 64, 1, ctypes.byref(e), L.CONV_FWD, 1, 16, 8, 64, 2,
                                    far, taps([0, 0]), None)
    assert rc != 0 and "tap offset out of range" in _error(lib)
    g = L.ConvGeom()
    g.mode, g.N, g.H, g.W, g.C, g.n_taps = L.CONV_FWD, 1, 16, 8, 64, 33
    rc = lib.pg_gemm_bf16_conv(p, 64, p, 64, 128, 64, 33 * 64, 1, ctypes.byref(e), ctypes.byref(g), None)
    assert rc != 0 and "1..32 taps in a pg_conv_geom (got 33)" in _error(lib)
    for name in ("pg_tap_gather", "pg_tap_scatter"):
        if name == "pg_tap_gather":
            rc = lib.pg_tap_gather(p, 8, 1, 4, 4, 8, 226, z226, z226, 0, p, None)
        else:
            rc = lib.pg_tap_scatter(p, 1, 4, 4, 8, 226, z226, z226, 0, None, 0, p, None, 8, None)
        assert rc != 0 and "226 taps (max 225)" in _error(lib), name
    rc = lib.pg_conv_small_fwd_d(p, p, None, 1, 3, 4, 4, 8, 3, 3, 1, 1, 0, 1, 0, p, None, 0, None)
    assert rc != 0 and "dilation (0, 1) must be positive" in _error(lib)
    rc = lib.pg_conv_small_bwd_d(p, p, p, 1, 3, 4, 4, 8, 3, 3, 1, 1, 1, -2, 0, p, None, None, None)
    assert rc != 0 and "dilation (1, -2) must be positive" in _error(lib)


def _forward_on_cpu(monkeypatch, m):
    """CausalConv2d.forward up to the CUDA path: the argument checks run, then the path refuses the CPU tensor."""
    from pytorch_generative_b200.nn import modules

    monkeypatch.setattr(modules, "_require_cuda", lambda x, who: None)
    return m(torch.zeros(1, m.in_channels, 8, 8))


@pytest.mark.parametrize("kwargs", [dict(stride=2), dict(groups=2), dict(padding_mode="reflect"),
                                    dict(padding=2), dict(dilation=2), dict(dilation=2, padding=3),
                                    dict(dilation=(2, 1), padding=(2, 2))],
                         ids=["stride", "groups", "padding_mode", "pad2", "dil2_pad1", "dil2_pad3", "dil21_pad22"])
def test_causal_conv2d_arguments_off_the_path_still_raise(monkeypatch, kwargs):
    from pytorch_generative_b200 import nn

    kw = dict(padding=1)
    kw.update(kwargs)
    with pytest.raises(NotImplementedError):
        _forward_on_cpu(monkeypatch, nn.CausalConv2d(True, 4, 8, 3, **kw))


@pytest.mark.parametrize("k,kwargs", [(3, dict(padding=2, dilation=2)), (7, dict(padding=(6, 3), dilation=(2, 1))),
                                      (15, dict(padding=7)), ((3, 5), dict(padding=(3, 6), dilation=3))])
def test_causal_conv2d_takes_dilation_with_same_padding(monkeypatch, k, kwargs):
    """Dilation with padding d (k // 2) passes the argument checks and reaches the CUDA path (which refuses CPU
    tensors); the mask is built from kernel positions, unchanged by the dilation."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import nn

    m = nn.CausalConv2d(False, 4, 8, k, **kwargs)
    kh, kw = m.weight.shape[-2:]
    assert torch.equal(m.mask, O.causal_mask(kh, kw, False).expand_as(m.weight))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        _forward_on_cpu(monkeypatch, m)
