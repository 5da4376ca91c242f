"""ImageGPT's recompute path: the fused stack keeps only each block's input stream, attention output and lse, and
rebuilds the rest of a block's activations just before its backward.  It runs the same kernels on the same inputs as
the forward, so logits, loss and every gradient must be bit-identical to the path that keeps everything; only the
memory differs.  Each test forces the path by replacing models.image_gpt.recompute_activations."""

import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu

GAMMA = 0.999977

C2 = dict(in_channels=1, out_channels=1, in_size=28, n_transformer_blocks=8, n_attention_heads=4, n_embedding_channels=64)
C5_BLOCKS = dict(in_channels=3, out_channels=3, in_size=32, n_transformer_blocks=2, n_attention_heads=8,
                 n_embedding_channels=512)
HEAD_128 = dict(in_channels=3, out_channels=3, in_size=16, n_transformer_blocks=2, n_attention_heads=1,
                n_embedding_channels=128)
SIDE_64 = dict(in_channels=1, out_channels=1, in_size=64, n_transformer_blocks=2, n_attention_heads=2,
               n_embedding_channels=128)


def dev():
    return torch.device("cuda:0")


def _batch(n, cfg, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (n, cfg["in_channels"], cfg["in_size"], cfg["in_size"])
    if cfg["in_channels"] == 1:
        return torch.bernoulli(torch.full(shape, 0.5), generator=g)
    return torch.randint(0, 256, shape, generator=g).float() / 255


def _force(monkeypatch, recompute):
    """Makes the stack take one path; returns the decisions taken (the rule must never run under graph capture)."""
    from pytorch_generative_b200.models import image_gpt

    decisions = []

    def rule(mem, available):
        assert not torch.cuda.is_current_stream_capturing(), "the memory rule ran during CUDA-graph capture"
        decisions.append(recompute)
        return recompute

    monkeypatch.setattr(image_gpt, "recompute_activations", rule)
    return decisions


def _count_rebuilds(monkeypatch):
    from pytorch_generative_b200.models import image_gpt

    rebuilt = []
    block_fwd = image_gpt._block_fwd

    def counting(*args, attn=None, **kw):
        if attn is not None:
            rebuilt.append(1)
        return block_fwd(*args, attn=attn, **kw)

    monkeypatch.setattr(image_gpt, "_block_fwd", counting)
    return rebuilt


def _forward_backward(m, x):
    from pytorch_generative_b200 import losses

    m.zero_grad(set_to_none=True)
    xr = x.clone().requires_grad_(True)
    logits = m(xr)
    loss = losses.bce_with_logits_sum_mean(logits, x)
    loss.backward()
    out = dict(logits=logits.detach(), loss=loss.detach(), input_grad=xr.grad)
    out.update({name: p.grad for name, p in m.named_parameters()})
    assert all(v is not None for v in out.values())
    return out


@pytest.mark.parametrize("name,cfg,batch", [
    ("C2 geometry, padded head slots", C2, 4),
    ("C5 blocks", C5_BLOCKS, 2),
    ("one 128-channel head", HEAD_128, 2),
    ("64x64", SIDE_64, 2),
])
def test_recompute_is_bit_identical_to_store(monkeypatch, name, cfg, batch):
    from pytorch_generative_b200 import models

    torch.manual_seed(0)
    m = models.ImageGPT(**cfg).to(dev()).train()
    x = _batch(batch, cfg, seed=1).to(dev())
    rebuilt = _count_rebuilds(monkeypatch)
    _force(monkeypatch, False)
    stored = _forward_backward(m, x)
    assert not rebuilt
    _force(monkeypatch, True)
    recomputed = _forward_backward(m, x)
    assert len(rebuilt) == cfg["n_transformer_blocks"], "the backward did not rebuild every block"
    assert stored.keys() == recomputed.keys()
    for k in stored:
        assert torch.equal(stored[k], recomputed[k]), f"{name}: {k} differs between the store and recompute paths"


def test_graphed_recompute_trajectory_matches_eager_store(monkeypatch):
    """Three Adam steps: GraphedTrainStep with recompute forced (decided by its eager warm-up, reused by the capture)
    against the same arithmetic launched eagerly on the store path: loss, gradient norm and weights bit for bit."""
    from pytorch_generative_b200 import losses, models, trainstep

    cfg, lr = dict(in_channels=3, out_channels=3, in_size=16, n_transformer_blocks=2, n_attention_heads=2,
                   n_embedding_channels=128), 5e-3
    torch.manual_seed(0)
    init = {k: v.detach().clone() for k, v in models.ImageGPT(**cfg).state_dict().items()}
    xs = [_batch(4, cfg, seed=10 + i) for i in range(3)]
    loss_fn = lambda preds, x: losses.bce_with_logits_sum_mean(preds, x)  # noqa: E731

    def fresh():
        m = models.ImageGPT(**cfg)
        m.load_state_dict(init)
        return m.to(dev()).train()

    _force(monkeypatch, False)
    m = fresh()
    params = list(m.parameters())
    lr_t = torch.tensor(lr, device=dev())
    opt = torch.optim.Adam(params, lr=lr_t, capturable=True)  # GraphedTrainStep's step, launched eagerly
    ref = []
    for x in xs:
        xd = x.to(dev())
        opt.zero_grad(set_to_none=True)
        loss = loss_fn(m(xd), xd)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(params, 1e50, foreach=True)
        opt.step()
        lr_t.mul_(GAMMA)
        ref.append((loss.item(), norm.item()))
    ref_state = {k: v.detach().clone() for k, v in m.state_dict().items()}

    decisions = _force(monkeypatch, True)
    rebuilt = _count_rebuilds(monkeypatch)
    m = fresh()
    step = trainstep.GraphedTrainStep(m, list(m.parameters()), loss_fn, xs[0].to(dev()), lr=lr, lr_gamma=GAMMA)
    assert decisions and all(decisions) and rebuilt  # the eager warm-up took the recompute path
    n_rebuilt = len(rebuilt)
    step.reset(init)
    got = [step(x.to(dev())) for x in xs]
    assert len(rebuilt) == n_rebuilt  # replays launch the captured kernels, no Python
    assert got == ref
    for k, v in m.state_dict().items():
        assert torch.equal(v, ref_state[k]), k


def _activation_bytes(m, opt, x, monkeypatch, recompute):
    """(bytes held from forward to backward, peak bytes of forward + backward), both above what the step leaves behind:
    the weights, the optimizer state and the gradients."""
    from pytorch_generative_b200 import losses

    _force(monkeypatch, recompute)
    for _ in range(2):  # the first step warms up the allocator, the scratch buffers and the weight copies
        opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        loss = losses.bce_with_logits_sum_mean(m(x), x)
        kept = torch.cuda.memory_allocated() - base
        loss.backward()
        del loss
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - torch.cuda.memory_allocated()
        opt.clip_and_step(1e50)
    return kept, peak


@pytest.mark.parametrize("n_blocks,peak_ratio", [(8, 2.5), (24, 4.0)])
def test_recompute_shrinks_activation_memory(monkeypatch, n_blocks, peak_ratio):
    """512 channels, 8 heads, 32x32, batch 8.  Between forward and backward the recompute path keeps 3104 B per pixel and
    block against 18480: at least 4x less.  The peak also holds one block's rebuilt activations and its backward's
    gradient transients (about 25.6 KB per pixel at C = 512, whatever the depth), so its ratio approaches 6x with depth:
    about 3.0x at 8 blocks and 4.4x at 24 by activation_memory.  Both paths stay within that estimate."""
    from pytorch_generative_b200 import models, optim
    from pytorch_generative_b200.models import image_gpt

    cfg = dict(C5_BLOCKS, n_transformer_blocks=n_blocks)
    torch.manual_seed(0)
    m = models.ImageGPT(**cfg).to(dev()).train()
    opt = optim.FusedAdam(m.parameters(), lr=5e-3)
    x = _batch(8, cfg, seed=2).to(dev())
    kept_s, peak_s = _activation_bytes(m, opt, x, monkeypatch, False)
    kept_r, peak_r = _activation_bytes(m, opt, x, monkeypatch, True)
    est = image_gpt.activation_memory(8 * 32 * 32, 512, 8, 64, 64, n_blocks)
    print(f"{n_blocks} blocks: kept {kept_s / 2**20:.0f} / {kept_r / 2**20:.0f} MiB ({kept_s / kept_r:.2f}x), "
          f"peak {peak_s / 2**20:.0f} / {peak_r / 2**20:.0f} MiB ({peak_s / peak_r:.2f}x); estimate kept "
          f"{est.store / 2**20:.0f} / {est.recompute / 2**20:.0f} MiB, one block's backward {est.backward / 2**20:.0f} MiB")
    assert kept_s >= 4 * kept_r
    assert peak_s >= peak_ratio * peak_r
    assert 0.97 * est.store <= kept_s <= 1.03 * est.store
    assert 0.97 * est.recompute <= kept_r <= 1.03 * est.recompute
    assert peak_s <= est.store + est.backward
    assert peak_r <= est.recompute + est.store_block - est.recompute_block + est.backward


# --------------------------------------------------------------------------------------------------
# Data parallelism: the overlapped bucket hook sees the same gradient arena on both paths
# --------------------------------------------------------------------------------------------------
DP_CFG = dict(in_channels=3, out_channels=3, in_size=16, n_transformer_blocks=2, n_attention_heads=8,
              n_embedding_channels=512)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    from pytorch_generative_b200 import losses, models, parallel
    from pytorch_generative_b200.models import image_gpt

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    device = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    torch.manual_seed(0)
    m = models.ImageGPT(**DP_CFG).to(device)
    avg = parallel.OverlappedGradAverager(m)
    assert avg.n_bucketed == 2 * 5
    x = _batch(2, DP_CFG, seed=100 + rank).to(device)
    out = {}
    for recompute in (False, True):
        image_gpt.recompute_activations = lambda mem, available, r=recompute: r
        m.zero_grad(set_to_none=True)
        losses.bce_with_logits_sum_mean(m(x), x).backward()
        avg.average_()
        out[recompute] = {k: p.grad.detach().cpu() for k, p in m.named_parameters()}
    torch.save(out, os.path.join(out_dir, f"grads_{rank}.pt"))
    avg.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_overlapped_grad_averaging_is_identical_on_both_paths(tmp_path):
    import torch.multiprocessing as mp

    world = 2
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    grads = [torch.load(tmp_path / f"grads_{r}.pt") for r in range(world)]
    for k in grads[0][False]:
        for r in range(world):
            assert torch.equal(grads[r][False][k], grads[r][True][k]), f"rank {r}, {k}: paths differ after averaging"
        assert torch.equal(grads[0][True][k], grads[1][True][k]), f"{k}: ranks disagree after averaging"
