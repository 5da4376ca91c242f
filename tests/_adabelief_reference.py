"""Float64 restatement of the AdaBelief step (pg_adabelief_step, optim.AdaBelief) with per-element bounds, its bug
models, the inputs of the tests/golden/adabelief_rezero.pt trajectory and its packed tensors, and the bound of ReZero's alpha gradient.
Shared by tests/test_adabelief_rezero_cpu.py, tests/test_adabelief_rezero_gpu.py and
tests/golden/make_adabelief_rezero_golden.py; not a test module.

The step, per element, every operation rounded to fp32 in this order (the reference's optim.py with its tuple unpack
corrected), from the fp32 scalars pg_adabelief_step derives from the host's doubles:
    g' = g c,  c = min(1, max_norm / (norm + 1e-6))
    m' = b1 m + (1 - b1) g';  e = g' - m';  v' = b2 v + (1 - b2) e^2 + 1e-10
    p' = p - lr ((m' / bc1) / (sqrt(v' / bc2) + 1e-10)),   bc = fp32(1 - b^t) computed in double.
The reference takes the kernel's own fp32 norm (or clip_grad_norm_'s, for the CPU fixture), so the norm's error stays
out of these bounds; tests/_step_reference.sqnorm_reference bounds the norm itself.

Bounds (U = 2^-24; an fp32 operation costs U of the magnitude it produces, a product of rounded operands the sum of
their relative errors):
    g':  3 U |g'| when clipping (the coefficient's 2 U and the product's U), exact otherwise;
    m':  (1 - b1) b_g + 2 U (b1 |m| + (1 - b1) |g'|) + U |m'|;
    e:   (b_g + b_m)(1 + U) + U |e|.  e = g' - m' can cancel, so its bound scales with |g'| + |m'| through b_g and b_m,
         not with |e|;
    v':  (1 - b2) b_e2 (1 + 2 U) + 2 U (b2 v + (1 - b2) e^2) + 2 U v',  b_e2 = (2 |e| + b_e) b_e + U (|e| + b_e)^2;
    v' / bc2, sqrt, + 1e-10, the two divisions and the final subtraction: one U each on what they produce, the sqrt
         halving the relative error it takes in.
v' >= 1e-10 > 0 on every step (the stored variance takes the 1e-10 every time), so no relative error divides by 0."""

import math

import torch

from _step_reference import chunk_table, sqnorm_reference  # noqa: F401  (re-exported for the tests)

F64, F32 = torch.float64, torch.float32
U24 = 2.0 ** -24
EPS10 = float(torch.tensor(1e-10, dtype=F32))
EPS6 = float(torch.tensor(1e-6, dtype=F32))


def f32(v):
    return float(torch.tensor(v, dtype=F32))


def scalars(lr, beta1, beta2, step):
    """The fp32 scalars pg_adabelief_step hands its kernel, rounded as it rounds them."""
    return dict(lr=f32(lr), beta1=f32(beta1), beta2=f32(beta2), omb1=f32(1.0 - beta1), omb2=f32(1.0 - beta2),
                bc1=f32(1.0 - math.pow(beta1, step)), bc2=f32(1.0 - math.pow(beta2, step)))


BUGS = ("eps_once", "old_m", "adam_bc2", "unclipped", "lr_is_beta2")


def reference(p, g, m, v, norm, max_norm, sc, bug=None):
    """Float64 AdaBelief step of one tensor from fp32 p, g, m, v, the fp32 norm and the scalars `sc` (`scalars`).
    Returns dict p, g (after clipping), m, v and their bounds b_p, b_g, b_m, b_v.  `bug` selects a bug model:
      eps_once     the 1e-10 is not added to the stored variance (only the denominator's 1e-10 remains);
      old_m        e is taken from the old m;
      adam_bc2     the variance is divided by sqrt(bc2), Adam's correction of sqrt(v), instead of bc2;
      unclipped    the moments are fed the gradient before clipping;
      lr_is_beta2  the unpack "fixed" as `beta1, lr = group["betas"]`: the step size is beta2."""
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    coef = max_norm / (float(norm) + EPS6)
    clips = coef < 1.0
    coef = min(coef, 1.0)
    g1 = g64 * coef
    b_g = 3 * U24 * g1.abs() if clips else torch.zeros_like(g1)
    gm = g64 if bug == "unclipped" else g1
    b1, b2, o1, o2 = sc["beta1"], sc["beta2"], sc["omb1"], sc["omb2"]
    m1 = b1 * m64 + o1 * gm
    b_m = o1 * b_g + 2 * U24 * (b1 * m64.abs() + o1 * gm.abs()) + U24 * m1.abs()
    e = gm - (m64 if bug == "old_m" else m1)
    b_e = (b_g + b_m) * (1 + U24) + U24 * e.abs()
    e2 = e * e
    b_e2 = (2 * e.abs() + b_e) * b_e + U24 * (e.abs() + b_e) ** 2
    v1 = b2 * v64 + o2 * e2 + (0.0 if bug == "eps_once" else EPS10)
    b_v = o2 * b_e2 * (1 + 2 * U24) + 2 * U24 * (b2 * v64 + o2 * e2) + 2 * U24 * v1
    bc2 = math.sqrt(sc["bc2"]) if bug == "adam_bc2" else sc["bc2"]
    vh = v1 / bc2
    r_vh = b_v / v1.clamp_min(1e-300) + U24
    s = vh.sqrt()
    r_s = r_vh / 2 + r_vh ** 2 + U24
    d = s + EPS10
    r_d = r_s * s / d + U24
    mh = m1 / sc["bc1"]
    b_mh = b_m / sc["bc1"] + U24 * mh.abs()
    q = mh / d
    b_q = (b_mh + mh.abs() * (r_d + r_d ** 2)) / d + 2 * U24 * q.abs()
    lr = sc["beta2"] if bug == "lr_is_beta2" else sc["lr"]
    p1 = p64 - lr * q
    b_p = lr * (b_q + 2 * U24 * q.abs()) + U24 * (p1.abs() + lr * q.abs())
    return dict(p=p1, g=g1, m=m1, v=v1, b_p=b_p, b_g=b_g, b_m=b_m, b_v=b_v)


# ----------------------------------------------------------------------------------------------------------------------
# the fixture trajectory (tests/golden/adabelief_rezero.pt)
# ----------------------------------------------------------------------------------------------------------------------
# parameter name -> numel.  `none` never gets a gradient; `zero` always gets an all-zero one and `const` a constant one
# (the regimes where the 1e-10 added to the stored variance dominates it).
SIZES = {"a": 1, "b": 3, "c": 4097, "none": 5, "big": 70000, "zero": 8, "const": 6}
GROUPS = (dict(names=("a", "b", "c", "none"), lr=1e-3, betas=(0.9, 0.999)),
          dict(names=("big", "zero", "const"), lr=3e-3, betas=(0.8, 0.99)))
STEPS = 6
CLIP_STEPS = (2, 5)  # 1-based steps run with max_norm = CLIP_FRACTION x the gradient norm
CLIP_FRACTION = 0.5
GRAD_SCALES = (1.0, 0.1, 3.0, 1e-3, 1.0, 0.5)
# Initial values and gradients repeat with this period (a prime: the pattern crosses float4 and chunk boundaries at
# every phase).  Once the norm is fixed the step is elementwise, so each recorded tensor is its first PERIOD elements
# tiled, except where the reference's CPU loops round differently (their scalar tails): `pack` stores those positions
# explicitly and `unpack` rebuilds the tensor bit for bit.
PERIOD = 257


def _tiled(pattern, n):
    return pattern[torch.arange(n) % pattern.numel()]


def initial_params():
    g = torch.Generator().manual_seed(7)
    return {k: _tiled(torch.randn(min(n, PERIOD), generator=g), n) for k, n in SIZES.items()}


def grads_at(step):
    """Gradients of 1-based `step`: name -> fp32 tensor, or None for `none`."""
    g = torch.Generator().manual_seed(100 + step)
    out = {}
    for k, n in SIZES.items():
        if k == "none":
            out[k] = None
        elif k == "zero":
            out[k] = torch.zeros(n)
        elif k == "const":
            out[k] = torch.full((n,), 0.25)
        else:
            out[k] = _tiled(torch.randn(min(n, PERIOD), generator=g), n) * GRAD_SCALES[step - 1]
    return out


def pack(t):
    """A 1-D fp32 tensor as its first PERIOD elements and the positions where it differs from their tiling."""
    pattern = t[:PERIOD].clone()
    idx = torch.nonzero(_tiled(pattern, t.numel()).view(torch.int32) != t.view(torch.int32)).flatten()
    return dict(n=t.numel(), pattern=pattern, idx=idx.to(torch.int32), val=t[idx].clone())


def unpack(d):
    t = _tiled(d["pattern"], d["n"])
    t[d["idx"].long()] = d["val"]
    return t


def unpack_state_dict(sd):
    """A recorded optimizer state dict with its packed tensors rebuilt."""
    state = {i: {k: (unpack(v) if isinstance(v, dict) else v) for k, v in st.items()} for i, st in sd["state"].items()}
    return {"state": state, "param_groups": [dict(g) for g in sd["param_groups"]]}


def group_of(name):
    return next(gr for gr in GROUPS if name in gr["names"])


# ----------------------------------------------------------------------------------------------------------------------
# ReZero
# ----------------------------------------------------------------------------------------------------------------------
def dalpha_bound(dy, f):
    """(ref, bound) of sum(dy f) in float64.  Every term passes through at most d rounded additions, d the depth of
    pg_rezero_bwd's summation tree: a thread's chain over its PG_REZERO_CHUNK / 256 elements (plus one tail element),
    the warp butterfly (5), the butterfly over the block's 8 warp sums (5), pg_sum_partials' chain over the blocks
    (block count, or at 64 blocks and more a lane chain of ceil(blocks / 32) and a butterfly of 5) and the add onto
    dalpha (1).  The term's product adds one rounding and one more is spare: (d + 2) U sum|dy f|."""
    t = dy.to(F64).flatten() * f.to(F64).flatten()
    blocks = (t.numel() + 8191) // 8192
    depth = 8192 // 256 + 1 + 5 + 5 + ((blocks + 31) // 32 + 5 if blocks >= 64 else blocks) + 1
    return float(t.sum()), (depth + 2) * U24 * float(t.abs().sum())
