"""ImageGPT's choice between keeping every block's activations until backward and recomputing them
(models.image_gpt.activation_memory / recompute_activations), without a GPU."""

import pytest

C5 = dict(channels=512, n_heads=8, qk_slot=64, dv_slot=64, n_blocks=24)
GB = 1e9


def _estimate(batch, side, **kw):
    from pytorch_generative_b200.models import image_gpt

    return image_gpt.activation_memory(batch * side * side, **{**C5, **kw})


def test_store_path_keeps_about_1_2_gb_per_block_at_c5():
    """18480 B per pixel and block at C = 512 (xs, h fp32; a1, a2, o bf16; qkv bf16; u, g bf16 at 4C; LN statistics and
    lse), against 3104 B (xs, o, lse) on the recompute path."""
    small, large = _estimate(64, 32), _estimate(64, 64)
    assert small.store_block == 18480 * 64 * 32 * 32
    assert small.recompute_block == 3104 * 64 * 32 * 32
    assert 1.15 * GB < small.store_block < 1.25 * GB
    assert 4.8 * GB < large.store_block < 4.9 * GB
    assert 28 * GB < small.store < 30 * GB   # 24 blocks + the final stream and LayerNorm: DESIGN.md §3
    assert 116 * GB < large.store < 118 * GB
    assert 19.5 * GB < large.recompute < 21 * GB


def test_rule_keeps_everything_at_32x32_and_recomputes_at_64x64():
    from pytorch_generative_b200.models import image_gpt

    small, large = _estimate(64, 32), _estimate(64, 64)
    assert not image_gpt.recompute_activations(small, 75 * GB)
    assert image_gpt.recompute_activations(large, 75 * GB)
    # on the recompute path the 64x64 batch fits: kept activations, one block's rebuilt ones and its backward
    assert large.recompute + (large.store_block - large.recompute_block) + large.backward < 75 * GB


def test_rule_boundary_counts_one_block_backward():
    from pytorch_generative_b200.models import image_gpt

    m = _estimate(64, 32)
    assert not image_gpt.recompute_activations(m, m.store + m.backward)
    assert image_gpt.recompute_activations(m, m.store + m.backward - 1)
    assert image_gpt.recompute_activations(m, m.store)


def test_padded_head_slots_are_counted_at_slot_width():
    """C2 geometry: 4 heads of 16 channels live in 64-wide q/k and v slots, so qkv is 3 x 4 x 64 columns wide and the
    attention output 4 x 64, not 3 x 64 and 64."""
    from pytorch_generative_b200 import ops
    from pytorch_generative_b200.models import image_gpt

    C, H = 64, 4
    qk_slot, dv_slot = ops.head_slots(C // H, C // H)
    assert (qk_slot, dv_slot) == (64, 64)
    padded = image_gpt.activation_memory(1, C, H, qk_slot, dv_slot, 1)
    tight = image_gpt.activation_memory(1, C, H, C // H, C // H, 1)
    assert padded.store_block - tight.store_block == 2 * 3 * H * (64 - 16) + 2 * H * (64 - 16)
    assert padded.recompute_block - tight.recompute_block == 2 * H * (64 - 16)
    assert padded.store_block == 28 * C + 2 * 3 * H * 64 + 2 * H * 64 + 4 * H + 16
    assert padded.recompute_block == 4 * C + 2 * H * 64 + 4 * H


@pytest.mark.parametrize("batch,side", [(1, 8), (8, 28), (64, 32), (64, 64)])
def test_estimate_scales_with_pixels_and_blocks(batch, side):
    one, two = _estimate(batch, side, n_blocks=1), _estimate(batch, side, n_blocks=2)
    assert two.store - one.store == one.store_block
    assert two.recompute - one.recompute == one.recompute_block
    assert two.backward > one.backward  # the gradient arena grows with the blocks
    assert one.recompute_block * 5 < one.store_block
