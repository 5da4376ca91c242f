"""The layouts ImageGPT's fused backward writes through, without a GPU: the gradient arena (models.image_gpt.GradArena)
hands out disjoint views that cover its buffer, its buckets are the blocks' matrices, its size is the one
activation_memory counts, and BlockParams names the parameters in the order TransformerBlock lists them."""

import pytest
import torch

MATRICES = ("dw2", "dw1", "dwp", "dwqkv")
GEOMETRIES = [(512, 8), (512, 4), (64, 4), (96, 2), (12, 3), (15, 3), (100, 4)]


def _arena(c, heads, n_blocks):
    from pytorch_generative_b200.models import image_gpt
    from pytorch_generative_b200.nn.modules import head_layout

    sl, lay = image_gpt.stream_layout(c), head_layout(heads, c, c)
    return image_gpt.GradArena(n_blocks, sl, lay, torch.device("cpu")), sl, lay


def _span(buf, view):
    """[first, last + 1) of a contiguous view, in elements of buf."""
    assert view.is_contiguous() and view.dtype == buf.dtype
    first = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    return first, first + view.numel()


@pytest.mark.parametrize("n_blocks", [1, 2, 3])
@pytest.mark.parametrize("c,heads", GEOMETRIES)
def test_views_are_disjoint_and_cover_the_buffer(c, heads, n_blocks):
    from pytorch_generative_b200.models import image_gpt

    arena, sl, lay = _arena(c, heads, n_blocks)
    buf = arena.buf
    assert buf.dtype == torch.float32 and buf.dim() == 1 and not buf.any()
    assert buf.numel() == image_gpt.GradArena.numel(n_blocks, sl, lay)
    qkv_rows = heads * (2 * lay.qk_slot + lay.dv_slot)
    shapes = dict(dw2=(sl.c_p, sl.f_p), dw1=(sl.f_p, sl.c_p), dwp=(sl.c_p, heads * lay.dv_slot),
                  dwqkv=(qkv_rows, sl.c_p), ln1_stats=(3, c), ln2_stats=(3, c), dbqkv=(qkv_rows,), db1=(sl.f_p,))
    covered = torch.zeros(buf.numel(), dtype=torch.int32)
    for b in range(n_blocks):
        views = arena.block(b)
        assert views._fields == tuple(shapes)
        for name, view in zip(views._fields, views):
            assert tuple(view.shape) == shapes[name], (b, name)
            lo, hi = _span(buf, view)
            assert 0 <= lo and hi <= buf.numel(), (b, name)
            covered[lo:hi] += 1
    assert (covered == 1).all(), "two views overlap, or an element of the buffer belongs to none"
    # the matrices of every block, and nothing else, are the whole-stack bucket
    lo, hi = _span(buf, arena.bucket(0, n_blocks))
    small = [v for b in range(n_blocks) for n, v in zip(arena.block(b)._fields, arena.block(b)) if n not in MATRICES]
    assert lo == 0 and hi + sum(v.numel() for v in small) == buf.numel()
    assert all(_span(buf, v)[0] >= hi for v in small)


@pytest.mark.parametrize("c,heads", GEOMETRIES)
def test_bucket_holds_exactly_the_matrices_of_its_blocks(c, heads):
    n_blocks = 3
    arena, _, _ = _arena(c, heads, n_blocks)
    for lo in range(n_blocks):
        for hi in range(lo + 1, n_blocks + 1):
            first, last = _span(arena.buf, arena.bucket(lo, hi))
            inside = {(b, name) for b in range(n_blocks) for name, v in zip(arena.block(b)._fields, arena.block(b))
                      if first <= _span(arena.buf, v)[0] and _span(arena.buf, v)[1] <= last}
            assert inside == {(b, name) for b in range(lo, hi) for name in MATRICES}
            assert last - first == sum(getattr(arena.block(b), name).numel() for b, name in inside)


@pytest.mark.parametrize("n_blocks", [1, 2, 3])
@pytest.mark.parametrize("c,heads", [(512, 8), (512, 4)])
def test_identity_layouts_match_the_memory_estimate_and_give_views(c, heads, n_blocks):
    """Where neither heads nor stream are padded, the arena is what activation_memory counts, and the gradients handed
    to autograd share the arena's storage: an all-reduce of a bucket averages them in place (bucketed_parameters)."""
    from pytorch_generative_b200.models import image_gpt

    arena, sl, lay = _arena(c, heads, n_blocks)
    assert sl.identity and lay.identity and arena.views_are_grads
    est = image_gpt.activation_memory(0, c, heads, lay.qk_slot, lay.dv_slot, n_blocks)
    assert 4 * image_gpt.GradArena.numel(n_blocks, sl, lay) == est.backward
    storage = arena.buf.untyped_storage().data_ptr()
    for b in range(n_blocks):
        g = arena.block(b)
        nq = heads * lay.qk_slot
        grads = lay.unpack_grads(g.dwqkv[:nq], g.dbqkv[:nq], g.dwqkv[nq:], g.dbqkv[nq:], g.dwp, c, c)
        grads += (sl.unpack(g.dw1, (4 * c, c, 1, 1)), sl.unpack(g.db1, (4 * c,)), sl.unpack(g.dw2, (c, 4 * c, 1, 1)))
        assert [tuple(t.shape) for t in grads] == [(c, c, 1, 1), (c,), (2 * c, c, 1, 1), (2 * c,), (c, c, 1, 1),
                                                   (4 * c, c, 1, 1), (4 * c,), (c, 4 * c, 1, 1)]
        assert all(t.untyped_storage().data_ptr() == storage for t in grads)


def test_padded_geometries_do_not_offer_buckets():
    for c, heads in [(64, 4), (12, 3), (100, 4)]:
        assert not _arena(c, heads, 2)[0].views_are_grads
    assert not _arena(512, 8, 0)[0].views_are_grads


def test_block_params_name_the_parameters_in_flat_order():
    from pytorch_generative_b200.models import image_gpt

    blk = image_gpt.TransformerBlock(16, 2)
    a = blk._attn
    expected = [("ln1_w", blk._ln1.weight), ("ln1_b", blk._ln1.bias), ("q_w", a._q.weight), ("q_b", a._q.bias),
                ("kv_w", a._kv.weight), ("kv_b", a._kv.bias), ("p_w", a._proj.weight), ("p_b", a._proj.bias),
                ("ln2_w", blk._ln2.weight), ("ln2_b", blk._ln2.bias), ("f1_w", blk._out[0].weight),
                ("f1_b", blk._out[0].bias), ("f2_w", blk._out[2].weight), ("f2_b", blk._out[2].bias)]
    flat = blk.flat_params()
    assert isinstance(flat, image_gpt.BlockParams) and image_gpt.PARAMS_PER_BLOCK == len(expected) == len(flat)
    assert flat._fields == tuple(name for name, _ in expected)
    assert [t.data_ptr() for t in flat] == [t.data_ptr() for _, t in expected]
    assert len({t.data_ptr() for t in flat}) == len(expected)
    stem, blocks, head = image_gpt._split_params(["pos", "in_w", "in_b", *flat, *flat, "ln_w", "ln_b", "out_w", "out_b"])
    assert (list(stem), list(head)) == (["pos", "in_w", "in_b"], ["ln_w", "ln_b", "out_w", "out_b"])
    assert len(blocks) == 2 and all(t is u for got in blocks for t, u in zip(got, flat, strict=True))
