"""The memo of the bf16 weight copies (ops.cached_copy), driven on CPU tensors with a counting build: when an entry is
reused, when it is rebuilt, and that it lives exactly as long as its Parameter."""

import copy
import gc
import os
import socket
import weakref

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


class Counting:
    """A `build` that records how often the memo called it; each call returns a new tensor."""

    def __init__(self):
        self.calls = 0

    def __call__(self):
        self.calls += 1
        return torch.full((2,), float(self.calls))


def _param(*shape):
    return torch.nn.Parameter(torch.randn(*shape))


def test_unchanged_sources_hit():
    from pytorch_generative_b200 import ops

    p, build = _param(4, 3), Counting()
    first = ops.cached_copy((p,), "k", build)
    assert ops.cached_copy((p,), "k", build) is first and build.calls == 1
    assert ops.cached_copy((p,), "k", build) is first and build.calls == 1


@pytest.mark.parametrize("change", ["no_grad_inplace", "increment_version", "data_replaced"])
def test_a_changed_source_misses(change):
    from pytorch_generative_b200 import ops

    p, build = _param(4, 3), Counting()
    first = ops.cached_copy((p,), "k", build)
    old = p.data
    if change == "no_grad_inplace":
        with torch.no_grad():
            p.add_(1)
    elif change == "increment_version":
        torch.autograd.graph.increment_version(p)
    else:
        p.data = old.clone()
    again = ops.cached_copy((p,), "k", build)
    assert build.calls == 2 and again is not first
    assert ops.cached_copy((p,), "k", build) is again and build.calls == 2


@pytest.mark.parametrize("which", [0, 1, 2])
def test_any_source_of_a_multi_source_entry_invalidates_it(which):
    from pytorch_generative_b200 import ops

    ps, build = [_param(3), _param(5, 2), _param(1)], Counting()
    ops.cached_copy(ps, "k", build)
    assert build.calls == 1
    torch.autograd.graph.increment_version(ps[which])
    ops.cached_copy(ps, "k", build)
    assert build.calls == 2
    other = list(ps)
    other[which] = _param(*ps[which].shape)  # another object in that place
    ops.cached_copy(other, "k", build)
    assert build.calls == 3


def test_keys_with_different_padding_or_positions_stay_apart():
    from pytorch_generative_b200 import ops

    p, build = _param(8, 4, 3, 3), Counting()
    keys = [("taps", 8, None), ("taps", 16, None), ("taps", 8, ((0, 0), (0, 1))), ("taps", 8, ((0, 0), (1, 0)))]
    copies = [ops.cached_copy((p,), k, build) for k in keys]
    assert build.calls == len(keys)
    for k, c in zip(keys, copies):
        assert ops.cached_copy((p,), k, build) is c
    assert build.calls == len(keys)


def test_causal_mask_keeps_the_entry():
    from pytorch_generative_b200 import ops
    from pytorch_generative_b200.nn import CausalConv2d

    conv, build = CausalConv2d(mask_center=True, in_channels=2, out_channels=4, kernel_size=3, padding=1), Counting()
    conv.apply_mask()
    first = ops.cached_copy((conv.weight,), "k", build)
    with torch.no_grad():
        conv.weight.add_(1)  # an optimizer step: the masked taps move too, and so does the version
    conv.apply_mask()
    second = ops.cached_copy((conv.weight,), "k", build)
    assert second is not first and build.calls == 2
    conv.apply_mask()  # nothing to re-zero: the entry stays valid
    assert ops.cached_copy((conv.weight,), "k", build) is second and build.calls == 2
    assert float(conv.weight.detach()[:, :, 1, 1:].abs().sum()) == 0.0


def test_an_entry_dies_with_its_parameter():
    from pytorch_generative_b200 import ops

    p = _param(4, 3)
    alive = weakref.ref(ops.cached_copy((p,), "k", Counting()))
    gc.collect()
    assert alive() is not None  # held by the memo while p lives
    n = len(ops._COPIES)
    del p
    gc.collect()
    assert alive() is None and len(ops._COPIES) == n - 1


def test_a_deep_copy_finds_no_entries():
    from pytorch_generative_b200 import models, ops

    m = models.PixelCNN(in_channels=1, out_channels=1, n_residual=1, residual_channels=8, head_channels=8)
    build = Counting()
    for p in m.parameters():
        ops.cached_copy((p,), "k", build)
    n = build.calls
    c = copy.deepcopy(m)
    assert not any(p in ops._COPIES for p in c.parameters())
    for p in c.parameters():
        ops.cached_copy((p,), "k", build)
    assert build.calls == 2 * n
    for p in m.parameters():
        ops.cached_copy((p,), "k", build)
    assert build.calls == 2 * n  # the original's entries are untouched


def _broadcast_worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pytorch_generative_b200 import ops, parallel

    torch.manual_seed(100 + rank)
    model = torch.nn.Linear(6, 5)
    build = Counting()
    for p in model.parameters():
        ops.cached_copy((p,), "k", build)
    before = [p._version for p in model.parameters()]
    parallel.broadcast_parameters(model)
    after = [p._version for p in model.parameters()]
    for p in model.parameters():
        ops.cached_copy((p,), "k", build)
    torch.save(dict(before=before, after=after, calls=build.calls, n=len(before)), os.path.join(out_dir, f"b{rank}.pt"))
    dist.destroy_process_group()


def test_broadcast_parameters_moves_versions(tmp_path):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    world, port = 2, s.getsockname()[1]
    s.close()
    mp.spawn(_broadcast_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    for rank in range(world):
        r = torch.load(tmp_path / f"b{rank}.pt")
        assert all(a > b for a, b in zip(r["after"], r["before"])), r
        assert r["calls"] == 2 * r["n"]  # every copy made before the broadcast missed after it
