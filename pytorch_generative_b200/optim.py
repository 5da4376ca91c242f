"""`FusedAdam`: torch.optim.Adam's arithmetic (no amsgrad, no weight decay — what every recipe of the reference builds,
e.g. image_gpt.py:155) with the gradient-norm / clipping step of the trainer (reference trainer.py:182-186) folded in:
`clip_and_step(max_norm)` is two kernels over all parameters (`pg_grad_sqnorm`, `pg_adam_step`).

The optimizer state has torch.optim.Adam's layout (`step`, `exp_avg`, `exp_avg_sq` per parameter, same param_groups keys),
so `state_dict()` / `load_state_dict()` interchange with a checkpoint written by the reference Trainer.
"""

import torch

from . import _lib as L

CHUNK = 1 << 16  # elements per block


def chunk_table(numel, device):
    """The work list of the multi-tensor kernels for tensors of `numel` elements each: (numel as int64 [T], one
    (tensor, chunk) int32 row per CHUNK elements of each tensor, the number of rows), the tensors on `device`."""
    chunks = [(t, c) for t, n in enumerate(numel) for c in range((n + CHUNK - 1) // CHUNK)]
    return (torch.tensor(numel, dtype=torch.int64, device=device),
            torch.tensor(chunks, dtype=torch.int32, device=device).contiguous(), len(chunks))


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False):
        if weight_decay != 0 or amsgrad:
            raise NotImplementedError("FusedAdam implements the recipes' Adam: weight_decay=0, amsgrad=False")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=0, amsgrad=False, maximize=False, foreach=None,
                        capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False)
        super().__init__(params, defaults)
        self._plan = {}

    # ---- chunk plan: static per (group, participating parameters) ----
    def _build_plan(self, gi, params):
        dev = params[0].device
        numel, chunks, n_chunks = chunk_table([p.numel() for p in params], dev)
        n_t = len(params)
        host_ptrs = torch.empty(4, n_t, dtype=torch.int64).pin_memory()
        plan = dict(
            key=tuple(p.data_ptr() for p in params), n_chunks=n_chunks, numel=numel, chunks=chunks,
            partials=torch.empty(n_chunks, dtype=torch.float32, device=dev),
            norm_out=torch.zeros(2, dtype=torch.float32, device=dev),
            host_ptrs=host_ptrs, host_np=host_ptrs.numpy(), dev_ptrs=torch.empty(4, n_t, dtype=torch.int64, device=dev))
        self._plan[gi] = plan
        return plan

    def _state_for(self, p):
        st = self.state[p]
        if len(st) == 0:
            st["step"] = torch.tensor(0.0, dtype=torch.float32)  # torch.optim.Adam's default: a CPU scalar tensor
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    @torch.no_grad()
    def clip_and_step(self, max_norm=float("inf"), skip_above=None):
        """Total gradient norm over every parameter, clip to `max_norm`, Adam update.  Returns the norm as a device
        scalar (read it with `.item()` like the result of `clip_grad_norm_`).  With `skip_above`, a step whose norm
        exceeds it, or is NaN, leaves parameters and moments untouched (the trainer's `skip_grad_norm`).  Without it a
        NaN norm makes every gradient, moment and parameter NaN, as clip_grad_norm_ + torch.optim.Adam do."""
        if len(self.param_groups) != 1:
            # the recipes use one group; several groups would each need the global norm first
            raise NotImplementedError("FusedAdam.clip_and_step supports a single parameter group")
        self._opt_called = True  # what lr_scheduler's wrapper of step() records (its "step() before optimizer.step()" check)
        group = self.param_groups[0]
        params = [p for p in group["params"] if p.grad is not None]
        if not params:
            return torch.zeros((), device=group["params"][0].device)
        for p in params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise RuntimeError("FusedAdam: parameters must be contiguous fp32 CUDA tensors (no CPU fallback)")
            if not p.grad.is_contiguous():
                p.grad = p.grad.contiguous()
        plan = self._plan.get(0)
        if plan is None or plan["key"] != tuple(p.data_ptr() for p in params):
            plan = self._build_plan(0, params)
        states = [self._state_for(p) for p in params]
        if states[0]["step"].is_cuda:  # a checkpoint mapped onto the device: keep the counters on the host
            for st in states:
                st["step"] = st["step"].cpu()
        hp = plan["host_ptrs"]
        hn = plan["host_np"]  # numpy view of the pinned table: one vectorised fill per row, not a tensor index per entry
        hn[1, :] = [p.grad.data_ptr() for p in params]
        if plan.get("static_ok") != plan["key"]:  # parameter / moment addresses only change with the parameter set
            hn[0, :] = [p.data_ptr() for p in params]
            hn[2, :] = [st["exp_avg"].data_ptr() for st in states]
            hn[3, :] = [st["exp_avg_sq"].data_ptr() for st in states]
            plan["static_ok"] = plan["key"]
        plan["dev_ptrs"].copy_(hp, non_blocking=True)
        dp = plan["dev_ptrs"]
        L.grad_sqnorm(dp[1], plan["numel"], plan["chunks"], plan["n_chunks"], CHUNK, plan["partials"])
        step = int(states[0]["step"].item()) + 1
        beta1, beta2 = group["betas"]
        L.adam_step(dp[0], dp[1], dp[2], dp[3], plan["numel"], plan["chunks"], plan["n_chunks"], CHUNK, plan["partials"],
                    float(min(max_norm, 3.0e38)), float(skip_above or 0.0), float(group["lr"]), beta1, beta2, group["eps"],
                    step, plan["norm_out"])
        # the kernel wrote the parameters (and, when clipping, the gradients) through raw pointers: tell autograd and
        # every version-keyed cache (the models' bf16 weight copies) that they changed
        torch.autograd.graph.increment_version(params)
        norm = plan["norm_out"][0]
        applied = True
        if skip_above:
            applied = bool(plan["norm_out"][1].item() > 0)
        if applied:
            for st in states:
                st["step"] += 1
        return norm

    @torch.no_grad()
    def step(self, closure=None):
        """Plain Adam step (no clipping): torch.optim.Optimizer interface."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.clip_and_step(float("inf"))
        return loss
