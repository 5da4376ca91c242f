"""`FusedAdam` and `AdaBelief`, the optimizers of the CUDA path.

`FusedAdam`: torch.optim.Adam's arithmetic (no amsgrad, no weight decay — what every recipe of the reference builds,
e.g. image_gpt.py:155) with the gradient-norm / clipping step of the trainer (reference trainer.py:182-186) folded in:
`clip_and_step(max_norm)` is two kernels over all parameters (`pg_grad_sqnorm`, `pg_adam_step`).

The optimizer state has torch.optim.Adam's layout (`step`, `exp_avg`, `exp_avg_sq` per parameter, same param_groups keys),
so `state_dict()` / `load_state_dict()` interchange with a checkpoint written by the reference Trainer.

`AdaBelief`: the reference's `pytorch_generative.optim.AdaBelief` (optim.py) with the same clip / skip step folded in:
`clip_and_step` is one `pg_grad_sqnorm` pass over every group's gradients plus one `pg_adabelief_step` launch per
parameter group.  Its state and param groups have the reference's layout.
"""

import math

import torch

from . import _lib as L

CHUNK = 1 << 16  # elements per block


def chunk_table(numel, device):
    """The work list of the multi-tensor kernels for tensors of `numel` elements each: (numel as int64 [T], one
    (tensor, chunk) int32 row per CHUNK elements of each tensor, the number of rows), the tensors on `device`."""
    chunks = [(t, c) for t, n in enumerate(numel) for c in range((n + CHUNK - 1) // CHUNK)]
    return (torch.tensor(numel, dtype=torch.int64, device=device),
            torch.tensor(chunks, dtype=torch.int32, device=device).contiguous(), len(chunks))


def _build_plan(params):
    """The static part of a multi-tensor step over `params` (one device): the chunk table, the norm partials, the
    [2] norm_out and a pinned [4, T] pointer table (parameters, gradients, first and second moments) with its device
    copy."""
    dev = params[0].device
    numel, chunks, n_chunks = chunk_table([p.numel() for p in params], dev)
    n_t = len(params)
    host_ptrs = torch.empty(4, n_t, dtype=torch.int64).pin_memory()
    return dict(
        key=tuple(p.data_ptr() for p in params), n_chunks=n_chunks, numel=numel, chunks=chunks,
        partials=torch.empty(n_chunks, dtype=torch.float32, device=dev),
        norm_out=torch.zeros(2, dtype=torch.float32, device=dev),
        host_ptrs=host_ptrs, host_np=host_ptrs.numpy(), dev_ptrs=torch.empty(4, n_t, dtype=torch.int64, device=dev))


def _device_pointers(plan, params, moments):
    """Fills the plan's pointer table (gradients every step; parameters and `moments`, a list of (m, v) per parameter,
    when the parameter set changed) and queues its copy to the device.  Returns the device table."""
    hn = plan["host_np"]  # numpy view of the pinned table: one vectorised fill per row, not a tensor index per entry
    hn[1, :] = [p.grad.data_ptr() for p in params]
    if plan.get("static_ok") != plan["key"]:  # parameter / moment addresses only change with the parameter set
        hn[0, :] = [p.data_ptr() for p in params]
        hn[2, :] = [m.data_ptr() for m, _ in moments]
        hn[3, :] = [v.data_ptr() for _, v in moments]
        plan["static_ok"] = plan["key"]
    plan["dev_ptrs"].copy_(plan["host_ptrs"], non_blocking=True)
    return plan["dev_ptrs"]


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
        plan = _build_plan(params)
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
        dp = _device_pointers(plan, params, [(st["exp_avg"], st["exp_avg_sq"]) for st in states])
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


class AdaBelief(torch.optim.Optimizer):
    """The AdaBelief algorithm (Zhuang et al. 2020, arXiv:2010.07468) as the reference implements it: Adam with the
    running second moment of the gradient replaced by the running variance of its error g - m, no weight decay and no
    AMSGrad.  Per parameter with a gradient, in fp32:

        m = b1 m + (1 - b1) g;  e = g - m;  v = b2 v + (1 - b2) e^2 + 1e-10
        p -= lr (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t)) + 1e-10)

    The 1e-10 enters the stored variance on every step, as in the reference.  Parameters must be contiguous fp32 CUDA
    tensors; parameters whose `.grad` is None are skipped and get no state.  The state of a parameter is
    `{"step": int, "ema_avg", "ema_var"}` and the param groups hold `lr` and `betas`: the reference's layout, so its
    state dicts load here and this optimizer's load there."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999)):
        if not 0 <= lr:
            raise AssertionError(f"Invalid learning rate: {lr}")
        if not 0 <= betas[0] < 1:
            raise AssertionError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0 <= betas[1] < 1:
            raise AssertionError(f"Invalid beta parameter at index 1: {betas[1]}")
        super().__init__(params, dict(lr=lr, betas=betas))
        self._plan = None

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._plan = None  # the moments are new tensors: the pointer table must be refilled

    def _segments(self):
        """[(group, step, params)]: the parameters with a gradient, group by group and, inside a group, by step count
        (one launch each; a group whose parameters all stepped together is one segment)."""
        segments = []
        for group in self.param_groups:
            by_step = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("AdaBelief does not support sparse gradients.")
                if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                    raise RuntimeError("AdaBelief: parameters must be contiguous fp32 CUDA tensors (no CPU fallback)")
                if not p.grad.is_contiguous():
                    p.grad = p.grad.contiguous()
                st = self.state.get(p)
                by_step.setdefault(st["step"] if st else 0, []).append(p)
            segments += [(group, step, ps) for step, ps in by_step.items()]
        return segments

    @torch.no_grad()
    def clip_and_step(self, max_norm=float("inf"), skip_above=None):
        """Total gradient norm over the parameters of every group, clip to `max_norm`, AdaBelief update: one norm
        launch plus one update launch per group, no host synchronisation unless `skip_above` is given.  Returns the norm
        as a device scalar (like the result of `clip_grad_norm_`).  With `skip_above`, a step whose norm exceeds it, or
        is NaN, leaves parameters, gradients and state exactly as they were (no state is created by a skipped first
        step).  Without it a NaN norm makes every gradient, moment and parameter NaN, as clip_grad_norm_ followed by
        the reference step does."""
        self._opt_called = True  # what lr_scheduler's wrapper of step() records
        segments = self._segments()
        if not segments:
            return torch.zeros((), device=self.param_groups[0]["params"][0].device)
        params = [p for _, _, ps in segments for p in ps]
        created = [p for p in params if p not in self.state or len(self.state[p]) == 0]
        for p in created:
            self.state[p] = {"step": 0, "ema_avg": torch.zeros_like(p), "ema_var": torch.zeros_like(p)}
        states = [self.state[p] for p in params]
        key = (tuple(p.data_ptr() for p in params), tuple(len(ps) for _, _, ps in segments))
        if self._plan is None or self._plan["segments"] != key:
            self._plan = _build_plan(params)
            self._plan["segments"] = key
        plan = self._plan
        dp = _device_pointers(plan, params, [(st["ema_avg"], st["ema_var"]) for st in states])
        L.grad_sqnorm(dp[1], plan["numel"], plan["chunks"], plan["n_chunks"], CHUNK, plan["partials"])
        clip = float(min(max_norm, 3.0e38))
        first = 0  # first chunk-table row of the segment
        for group, step, ps in segments:
            n = sum(math.ceil(p.numel() / CHUNK) for p in ps)
            beta1, beta2 = group["betas"]
            L.adabelief_step(dp[0], dp[1], dp[2], dp[3], plan["numel"], plan["chunks"][first:first + n], n, CHUNK,
                             plan["partials"], plan["n_chunks"], clip, float(skip_above or 0.0), float(group["lr"]),
                             float(beta1), float(beta2), step + 1, plan["norm_out"])
            first += n
        # the kernels wrote the parameters (and, when clipping, the gradients) through raw pointers: tell autograd and
        # every version-keyed cache (the models' bf16 weight copies) that they changed
        torch.autograd.graph.increment_version(params)
        applied = not skip_above or bool(plan["norm_out"][1].item() > 0)
        if applied:
            for st in states:
                st["step"] += 1
        elif created:
            for p in created:
                del self.state[p]
            self._plan = None  # the next step creates new moment tensors
        return plan["norm_out"][0]

    @torch.no_grad()
    def step(self, closure=None):
        """The reference's step (no clipping): torch.optim.Optimizer interface."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.clip_and_step(float("inf"))
        return loss
