"""The head-slot rule of the attention kernels (ops.head_slots) and the slot layout of the projection weights
(nn.modules.HeadLayout), without a GPU."""

import pytest
import torch


def test_head_slots_pick_the_smallest_kernel_slot_and_set_the_layout_identity():
    from pytorch_generative_b200 import ops
    from pytorch_generative_b200.nn.modules import head_layout

    assert ops.head_slots(64, 64) == (64, 64)
    assert ops.head_slots(16, 128) == (64, 128)
    assert ops.head_slots(128, 32) == (128, 64)
    assert ops.head_slots(96, 80) == (128, 128)
    assert ops.head_slots(65, 1) == (128, 64)
    assert head_layout(1, 128, 128).identity and head_layout(1, 64, 128).identity
    assert not head_layout(1, 96, 96).identity and not head_layout(1, 32, 64).identity


@pytest.mark.parametrize("dk,dv", [(129, 64), (64, 256), (256, 256)])
def test_head_slots_refuse_heads_wider_than_128(dk, dv):
    from pytorch_generative_b200 import ops

    with pytest.raises(NotImplementedError, match="128"):
        ops.head_slots(dk, dv)


def _shares_storage(view, buf):
    return view.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr()


@pytest.mark.parametrize("pad", [False, True])
@pytest.mark.parametrize("dv", [32, 64, 128])
@pytest.mark.parametrize("dk", [16, 64, 96, 128])
@pytest.mark.parametrize("n_heads", [1, 4, 8])
def test_head_layout_scatter_then_unpack_returns_the_weights(n_heads, dk, dv, pad):
    """Scattering the projections into slot layout and gathering them back, as the gradients are, gives the original
    weights and biases bit for bit; padded slot rows and input columns are zero.  Without input-column padding the
    buffers are passed as ImageGPT does, as the q and kv rows of one fused qkv buffer.  When heads fill their slots,
    everything gathered is a view of the buffers passed in."""
    from pytorch_generative_b200 import ops
    from pytorch_generative_b200.nn.modules import head_layout

    H, embed, out_ch = n_heads, n_heads * dk, n_heads * dv
    cin_q, cin_kv = (34, 37) if pad else (64, 64)
    cin_q_pad, cin_kv_pad = ops.round_up(cin_q, 8), ops.round_up(cin_kv, 8)
    g = torch.Generator().manual_seed(n_heads * 1000 + dk * 10 + dv)
    q_w, kv_w = torch.randn(embed, cin_q, 1, 1, generator=g), torch.randn(embed + out_ch, cin_kv, 1, 1, generator=g)
    q_b, kv_b = torch.randn(embed, generator=g), torch.randn(embed + out_ch, generator=g)
    p_w = torch.randn(out_ch, out_ch, 1, 1, generator=g)

    lay = head_layout(H, embed, out_ch)
    assert lay.identity == (dk in ops.KERNEL_SLOTS and dv in ops.KERNEL_SLOTS)
    assert (lay.dk, lay.dv, (lay.qk_slot, lay.dv_slot)) == (dk, dv, ops.head_slots(dk, dv))
    wq, bq, wkv, bkv, wp = lay.scatter(q_w, q_b, kv_w, kv_b, p_w, cin_q_pad, cin_kv_pad)
    assert wq.shape == (H * lay.qk_slot, cin_q_pad) and bq.shape == (H * lay.qk_slot,)
    assert wkv.shape == (H * (lay.qk_slot + lay.dv_slot), cin_kv_pad) and bkv.shape == wkv.shape[:1]
    assert wp.shape == (out_ch, H * lay.dv_slot)
    for packed, true in ((wq, q_w), (bq, q_b), (wkv, kv_w), (bkv, kv_b), (wp, p_w)):
        assert packed.dtype == torch.float32 and torch.count_nonzero(packed) == torch.count_nonzero(true)

    if pad:  # separate buffers, and a gradient of the output projection with padded rows below out_ch
        bufs = (wq.clone(), bq.clone(), wkv.clone(), bkv.clone(), torch.cat((wp, torch.zeros(8, wp.shape[1]))))
        owners = bufs
    else:
        dwqkv, dbqkv, dwp = torch.cat((wq, wkv)), torch.cat((bq, bkv)), wp.clone()
        n_q = H * lay.qk_slot
        bufs = (dwqkv[:n_q], dbqkv[:n_q], dwqkv[n_q:], dbqkv[n_q:], dwp)
        owners = (dwqkv, dbqkv, dwqkv, dbqkv, dwp)
    got = lay.unpack_grads(*bufs, cin_q, cin_kv)
    for name, t, true, owner in zip(("q_w", "q_b", "kv_w", "kv_b", "p_w"), got, (q_w, q_b, kv_w, kv_b, p_w), owners):
        assert t.shape == true.shape and torch.equal(t, true), name
        if lay.identity:
            assert _shares_storage(t, owner), f"{name} is a copy, not a view of the buffer passed in"
