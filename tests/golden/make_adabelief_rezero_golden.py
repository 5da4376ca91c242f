"""Generates tests/golden/adabelief_rezero.pt from the reference checkout's AdaBelief (optim.py) and ReZeroWrapper
(nn/utils.py), on the CPU in fp32.

    python tests/golden/make_adabelief_rezero_golden.py <path to the reference checkout>

Both classes are broken as shipped, so neither is used quite as is:
  * AdaBelief.step fails on `beta1, beta2, lr = group["betas"], group["lr"]`.  The reference module is parsed with
    `ast`; the one assignment in AdaBelief.step whose target is a 3-tuple and whose value is a 2-tuple becomes
    `(beta1, beta2), lr = ...`, and the result is compiled into a throwaway module.  Nothing else changes, and no
    reference text is stored.
  * ReZeroWrapper.__init__ never calls Module.__init__: the wrapper is built with __new__, Module.__init__ and then the
    reference __init__.

AdaBelief: the trajectory of tests/_adabelief_reference (SIZES, GROUPS, STEPS): the gradients of every step are set,
torch.nn.utils.clip_grad_norm_ runs over the parameters with a gradient (max_norm = CLIP_FRACTION x the norm on
CLIP_STEPS, inf otherwise; its norm and max_norm are recorded), then the reference step.  Every step records p,
ema_avg and ema_var of every stepped parameter and the per-parameter step count; the reference optimizer's state_dict()
and parameters are recorded at steps 0 and 3.  Every recorded tensor is stored packed (tests/_adabelief_reference.pack:
the initial values and gradients repeat with a short period), and the generator checks that unpacking gives back the
reference's tensor bit for bit.

ReZero: state-dict keys, shapes and the initial alpha; for a wrapped CausalConv2d (3x3, mask B), NCHWLayerNorm and
Sequential(Conv2d 1x1, ReLU) on a 2x16x8x8 input: the module's state, x, the cotangent c, and at alpha = 0 and
alpha = ALPHA the output and the gradients of sum(y c) with respect to x, alpha and every module parameter.
"""

import ast
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _adabelief_reference as R  # noqa: E402

ALPHA = -0.375


def fixed_adabelief(reference):
    path = os.path.join(reference, "pytorch_generative", "optim.py")
    tree = ast.parse(open(path).read(), path)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "AdaBelief")
    step = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "step")
    hits = [n for n in ast.walk(step) if isinstance(n, ast.Assign) and len(n.targets) == 1
            and isinstance(n.targets[0], ast.Tuple) and len(n.targets[0].elts) == 3
            and isinstance(n.value, ast.Tuple) and len(n.value.elts) == 2]
    assert len(hits) == 1, f"expected one 3-from-2 tuple assignment in AdaBelief.step, found {len(hits)}"
    target = hits[0].targets[0]
    target.elts = [ast.Tuple(elts=target.elts[:2], ctx=ast.Store()), target.elts[2]]
    ast.fix_missing_locations(tree)
    ns = {"__name__": "adabelief_fixed"}
    exec(compile(tree, "<reference optim.py, unpack corrected>", "exec"), ns)
    return ns["AdaBelief"]


def packed(t):
    d = R.pack(t.detach())
    assert torch.equal(R.unpack(d).view(torch.int32), t.detach().view(torch.int32)), "packing lost bits"
    assert d["idx"].numel() <= 512, f"{d['idx'].numel()} positions differ from the tiled pattern"
    return d


def packed_state_dict(sd):
    out = {"state": {}, "param_groups": [dict(g) for g in sd["param_groups"]]}
    for k, st in sd["state"].items():
        out["state"][k] = {n: (packed(v) if torch.is_tensor(v) else v) for n, v in st.items()}
    return out


def adabelief_trajectory(AdaBelief):
    init = R.initial_params()
    params = {k: torch.nn.Parameter(v.clone()) for k, v in init.items()}
    groups = [dict(params=[params[n] for n in gr["names"]], lr=gr["lr"], betas=gr["betas"]) for gr in R.GROUPS]
    opt = AdaBelief(groups)
    state_dicts = {0: packed_state_dict(opt.state_dict())}
    steps = []
    for t in range(1, R.STEPS + 1):
        grads = R.grads_at(t)
        for k, p in params.items():
            p.grad = None if grads[k] is None else grads[k].clone()
        stepped = [p for p in params.values() if p.grad is not None]
        max_norm = float("inf")
        if t in R.CLIP_STEPS:
            max_norm = R.CLIP_FRACTION * float(torch.linalg.vector_norm(torch.cat([p.grad for p in stepped])))
        norm = torch.nn.utils.clip_grad_norm_(stepped, max_norm)
        opt.step()
        rec = dict(max_norm=max_norm, norm=float(norm), p={}, m={}, v={}, step={})
        for k, p in params.items():
            if k == "none":
                assert p not in opt.state or not opt.state[p], "a parameter without gradient got state"
                continue
            st = opt.state[p]
            rec["p"][k] = packed(p)
            rec["m"][k] = packed(st["ema_avg"])
            rec["v"][k] = packed(st["ema_var"])
            rec["step"][k] = st["step"]
        steps.append(rec)
        if t == 3:
            state_dicts[3] = packed_state_dict(opt.state_dict())
            state_dicts["params_3"] = {k: packed(p) for k, p in params.items()}
    return dict(steps=steps, state_dicts=state_dicts)


def rezero_cases(reference):
    from pytorch_generative.nn.convolution import CausalConv2d, NCHWLayerNorm
    from pytorch_generative.nn.utils import ReZeroWrapper

    def wrap(module):
        w = ReZeroWrapper.__new__(ReZeroWrapper)
        torch.nn.Module.__init__(w)
        ReZeroWrapper.__init__(w, module)
        return w

    torch.manual_seed(0)
    modules = dict(conv=CausalConv2d(False, 16, 16, 3, padding=1), ln=NCHWLayerNorm(16),
                   seq=torch.nn.Sequential(torch.nn.Conv2d(16, 16, 1), torch.nn.ReLU()))
    with torch.no_grad():  # a LayerNorm away from its (1, 0) initialisation
        modules["ln"].weight.copy_(torch.rand(16) + 0.5)
        modules["ln"].bias.copy_(torch.randn(16) * 0.1)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 16, 8, 8, generator=g)
    c = torch.randn(2, 16, 8, 8, generator=g)
    cases = {}
    for name, module in modules.items():
        w = wrap(module)
        sd = w.state_dict()
        case = dict(keys=list(sd), shapes={k: tuple(v.shape) for k, v in sd.items()},
                    alpha0=w._alpha.detach().clone(), state={k: v.clone() for k, v in sd.items()})
        for alpha in (0.0, ALPHA):
            w.load_state_dict(case["state"])
            with torch.no_grad():
                w._alpha.fill_(alpha)
            w.zero_grad()
            xs = x.clone().requires_grad_(True)
            y = w(xs)
            (y * c).sum().backward()
            case[alpha] = dict(y=y.detach().clone(), dx=xs.grad.clone(), dalpha=w._alpha.grad.clone(),
                               grads={k: p.grad.clone() for k, p in w._module.named_parameters()})
        cases[name] = case
    return dict(x=x, c=c, alpha=ALPHA, cases=cases)


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    out = dict(adabelief=adabelief_trajectory(fixed_adabelief(reference)), rezero=rezero_cases(reference))
    torch.save(out, os.path.join(HERE, "adabelief_rezero.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
