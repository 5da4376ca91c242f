"""The head-slot rule of the attention kernels (ops.head_slots), without a GPU."""

import pytest


def test_head_slots_pick_the_smallest_kernel_slot():
    from pytorch_generative_b200 import ops

    assert ops.head_slots(64, 64) == (64, 64)
    assert ops.head_slots(16, 128) == (64, 128)
    assert ops.head_slots(128, 32) == (128, 64)
    assert ops.head_slots(96, 80) == (128, 128)
    assert ops.head_slots(65, 1) == (128, 64)
    assert ops.heads_fill_slots(128, 128) and ops.heads_fill_slots(64, 128)
    assert not ops.heads_fill_slots(96, 96) and not ops.heads_fill_slots(32, 64)


@pytest.mark.parametrize("dk,dv", [(129, 64), (64, 256), (256, 256)])
def test_head_slots_refuse_heads_wider_than_128(dk, dv):
    from pytorch_generative_b200 import ops

    with pytest.raises(NotImplementedError, match="128"):
        ops.head_slots(dk, dv)
