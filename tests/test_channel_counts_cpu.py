"""Channel counts that are not multiples of 8, without a GPU: ImageGPT builds the reference's parameters at any width,
and the padded stream layout of its fused stack (models.image_gpt.StreamLayout) packs and unpacks weights exactly."""

import pytest
import torch


@pytest.mark.parametrize("c,heads", [(4, 2), (12, 3), (20, 4), (100, 4)])
def test_image_gpt_builds_the_reference_state_at_any_width(c, heads):
    from oracle import reference_path as O
    from pytorch_generative_b200 import models

    cfg = dict(in_channels=1, out_channels=1, in_size=8, n_transformer_blocks=2, n_attention_heads=heads,
               n_embedding_channels=c)
    m = models.ImageGPT(**cfg)
    ref = O.init_state("image_gpt", cfg)
    got = m.state_dict()
    assert set(got) == set(ref)
    for k, v in ref.items():
        assert got[k].shape == v.shape, k


@pytest.mark.parametrize("c", [1, 4, 12, 16, 20, 100])
def test_stream_layout_pack_then_unpack_returns_the_weights(c):
    """Every parameter of a block padded into the stream layout and cropped back, as its gradient is, gives the
    original bits; pad rows, columns and bias entries are zero.  At c % 8 == 0 nothing is copied."""
    from pytorch_generative_b200.models.image_gpt import stream_layout

    sl = stream_layout(c)
    assert (sl.c, sl.c_p % 8, sl.f_p % 8) == (c, 0, 0) and sl.c_p - c < 8 and sl.f_p - 4 * c < 8
    assert sl.identity == (c % 8 == 0)
    g = torch.Generator().manual_seed(c)
    params = {  # shape, packed rows, packed columns (None: a bias)
        "in_w": ((c, 3, 3, 3), sl.c_p, 27),
        "in_b": ((c,), sl.c_p, None),
        "proj_b": ((c,), sl.c_p, None),
        "fc1_w": ((4 * c, c, 1, 1), sl.f_p, sl.c_p),
        "fc1_b": ((4 * c,), sl.f_p, None),
        "fc2_w": ((c, 4 * c, 1, 1), sl.c_p, sl.f_p),
        "fc2_b": ((c,), sl.c_p, None),
    }
    for name, (shape, rows, cols) in params.items():
        w = torch.randn(shape, generator=g)
        packed = sl.pack(w, rows, cols)
        assert packed.dtype == torch.float32 and packed.shape == ((rows,) if cols is None else (rows, cols)), name
        assert torch.count_nonzero(packed) == torch.count_nonzero(w), name
        lead = packed[: shape[0]] if cols is None else packed[: shape[0], : w[0].numel()]
        assert torch.equal(lead.reshape(shape), w), name
        back = sl.unpack(packed.clone(), shape)
        assert back.shape == w.shape and torch.equal(back, w), name
        if sl.identity:
            assert packed.data_ptr() == w.data_ptr(), f"{name}: copied although nothing is padded"
