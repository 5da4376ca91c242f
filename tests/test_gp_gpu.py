"""GaussianProcess on the H100: pg_gemm_f64, pg_gp_potrf and pg_gp_trsm against exact integer products and float64
bounds; the model against the reference's fixture (tests/golden/gp.pt) at condition-scaled bounds; conditioned-out
points, rank-deficient sampling, the Thompson loop, sampling statistics, determinism, launch counts, CUDA-graph capture
and a large case against float64 on the CPU.  fp64 bit-equality is checked on int64 views."""

import itertools
import math
import os

import pytest
import torch

import _gp_reference as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
U = 2.0 ** -53
NB = 64
SIZES = (1, 15, 16, 17, 127, 128, 129, 1000)


@pytest.fixture(scope="module")
def lib():
    from pytorch_generative_b200 import _build, _lib

    _build.build(verbose=False)
    _lib.load()
    return _lib


@pytest.fixture(scope="module")
def fixture():
    return torch.load(os.path.join(ROOT, "tests", "golden", "gp.pt"), weights_only=False)


def bits(t):
    return t.reshape(-1).contiguous().view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()])


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def same_integers(got, ref):
    """Bit-equality of integer-valued results; +0.0 and -0.0 are the same integer."""
    return same_bits(got + 0.0, ref + 0.0)


def ints(*shape, lo=-8, hi=9, g=None):
    return torch.randint(lo, hi, shape, generator=g).to(F64)


def op(t, trans):
    return t.T if trans else t


# ------------------------------------------------------------------------------------------------ pg_gemm_f64
def test_gemm_exact_on_integers(lib):
    g = torch.Generator().manual_seed(0)
    scalars = (0.0, 1.0, -1.0, 2.0)
    for i, (m, n, k) in enumerate(itertools.product(SIZES, SIZES, SIZES)):
        ta, tb = bool(i & 1), bool(i & 2)
        alpha, beta = scalars[i % 4], scalars[(i // 4) % 4]
        A = ints(*((k, m) if ta else (m, k)), g=g)
        B = ints(*((n, k) if tb else (k, n)), g=g)
        C = ints(m, n, g=g)
        ref = alpha * (op(A, ta) @ op(B, tb)) + beta * C
        got = lib.gemm_f64(A.cuda(), B.cuda(), C.cuda(), trans_a=ta, trans_b=tb, alpha=alpha, beta=beta).cpu()
        assert same_integers(got, ref), (m, n, k, ta, tb, alpha, beta)


def test_gemm_every_transpose_pair_and_scalar_at_tile_edges(lib):
    g = torch.Generator().manual_seed(1)
    for ta, tb, alpha, beta in itertools.product((False, True), (False, True), (0.0, 1.0, -1.0, 2.0),
                                                 (0.0, 1.0, -1.0, 2.0)):
        m, n, k = 129, 65, 47
        A = ints(*((k, m) if ta else (m, k)), g=g)
        B = ints(*((n, k) if tb else (k, n)), g=g)
        C = ints(m, n, g=g)
        ref = alpha * (op(A, ta) @ op(B, tb)) + beta * C
        got = lib.gemm_f64(A.cuda(), B.cuda(), C.cuda(), trans_a=ta, trans_b=tb, alpha=alpha, beta=beta).cpu()
        assert same_integers(got, ref), (ta, tb, alpha, beta)


def test_gemm_beta_zero_ignores_nan_in_c(lib):
    A, B = ints(33, 20), ints(20, 17)
    C = torch.full((33, 17), float("nan"), dtype=F64)
    assert same_integers(lib.gemm_f64(A.cuda(), B.cuda(), C.cuda()).cpu(), A @ B)


def test_gemm_lower_only_leaves_the_upper_triangle(lib):
    g = torch.Generator().manual_seed(2)
    for n, k in ((1, 3), (64, 16), (65, 17), (200, 64), (257, 5)):
        A = ints(n, k, g=g)
        C0 = ints(n, n, g=g)
        got = lib.gemm_f64(A.cuda(), A.cuda(), C0.clone().cuda(), trans_b=True, alpha=-1.0, beta=1.0,
                           lower_only=True).cpu()
        full = C0 - A @ A.T
        low = torch.tril(torch.ones(n, n, dtype=torch.bool))
        assert same_integers(got[low], full[low]) and same_bits(got[~low], C0[~low]), (n, k)


def test_gemm_random_within_float64_bounds(lib):
    g = torch.Generator().manual_seed(3)
    for m, n, k in ((1000, 129, 1000), (17, 1000, 513), (256, 256, 4096)):
        A, B = torch.randn(m, k, generator=g, dtype=F64), torch.randn(k, n, generator=g, dtype=F64)
        got = lib.gemm_f64(A.cuda(), B.cuda(), torch.empty(m, n, dtype=F64, device="cuda")).cpu()
        bound = k * 2.0 ** -52 * (A.abs() @ B.abs())
        assert ((got - A @ B).abs() <= bound).all(), (m, n, k)


def test_gemm_k_order_does_not_depend_on_m_n_or_the_tile(lib):
    g = torch.Generator().manual_seed(4)
    A, B = torch.randn(300, 777, generator=g, dtype=F64).cuda(), torch.randn(777, 200, generator=g, dtype=F64).cuda()
    full = lib.gemm_f64(A, B, torch.empty(300, 200, dtype=F64, device="cuda"))
    part = lib.gemm_f64(A[37:101].contiguous(), B[:, 5:70].contiguous(), torch.empty(64, 65, dtype=F64, device="cuda"))
    assert same_bits(part, full[37:101, 5:70])


# ------------------------------------------------------------------------------------------------ pg_gp_potrf
def int_factor(n, g, zero_cols=()):
    L = torch.tril(ints(n, n, lo=-3, hi=4, g=g), -1)
    L += torch.diag(2.0 ** torch.randint(0, 4, (n,), generator=g).to(F64))
    for j in zero_cols:
        L[j, :] = 0
        L[:, j] = 0
    return L


def potrf(lib, A, noise=0.0):
    d = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = lib.gp_potrf(A.clone().cuda(), noise, d).cpu()
    return out, int(d)


def test_potrf_exact_on_integer_factors_across_block_edges(lib):
    g = torch.Generator().manual_seed(5)
    for n in (1, 2, 63, 64, 65, 127, 128, 129, 200, 257):
        L = int_factor(n, g)
        A = L @ L.T
        A = A + torch.triu(torch.full_like(A, 7.0), 1)  # the strict upper triangle is ignored (zeroed)
        got, dropped = potrf(lib, A)
        assert same_integers(got, L) and dropped == 0, n


def test_potrf_drops_zero_columns_exactly(lib):
    g = torch.Generator().manual_seed(6)
    n, cols = 200, (0, 63, 64, 100, 199)
    L = int_factor(n, g, cols)
    got, dropped = potrf(lib, L @ L.T)
    assert dropped == len(cols) and same_integers(got, L)


def test_potrf_duplicated_point_is_dropped(lib):
    g = torch.Generator().manual_seed(7)
    x = torch.rand(90, 3, generator=g, dtype=F64) * 4
    x = torch.cat([x[:70], x[10:11], x[70:]])  # point 10 again at row 70
    K = R.SqExp(1.0, 0.5)(x, x).detach()
    got, dropped = potrf(lib, K)
    assert dropped == 1 and torch.all(got[:, 70] == 0)
    ref, ref_dropped = R.psd_cholesky(K)
    assert ref_dropped == 1
    assert ((got - ref).abs() <= 64 * 91 * U * (ref.abs() @ ref.abs().T).diagonal().sqrt()[:, None]).all()


def test_potrf_nan_pivot_propagates(lib):
    g = torch.Generator().manual_seed(8)
    B = torch.randn(100, 100, generator=g, dtype=F64)
    A = B @ B.T + 100 * torch.eye(100, dtype=F64)
    A[30, 30] = float("nan")
    got, dropped = potrf(lib, A)
    assert dropped == 0 and torch.isnan(got[30, 30]) and torch.isnan(got[31:, 30]).all()
    assert torch.isfinite(got[:30, :30]).all()


def test_potrf_backward_error_on_random_spd(lib):
    g = torch.Generator().manual_seed(9)
    for n, noise in ((65, 0.0), (300, 1e-3), (1000, 0.5)):
        B = torch.randn(n, n, generator=g, dtype=F64)
        A = B @ B.T / n + 1e-2 * torch.eye(n, dtype=F64)
        got, dropped = potrf(lib, A, noise)
        assert dropped == 0 and same_bits(got, torch.tril(got))
        An = A + noise * torch.eye(n, dtype=F64)
        bound = 2 * n * U * (got.abs() @ got.abs().T)
        assert ((An - got @ got.T).abs() <= bound).all(), n


# ------------------------------------------------------------------------------------------------ pg_gp_trsm
def test_trsm_exact_on_integer_systems(lib):
    g = torch.Generator().manual_seed(10)
    for n, ncols in ((1, 1), (64, 33), (65, 100), (200, 7), (257, 65)):
        L = int_factor(n, g)
        X = ints(n, ncols, g=g)
        for transpose in (False, True):
            B = (L.T if transpose else L) @ X
            got = lib.gp_trsm(L.cuda(), B.cuda(), transpose=transpose).cpu()
            assert same_integers(got, X), (n, ncols, transpose)


def test_trsm_zero_diagonal_gives_zero_rows(lib):
    g = torch.Generator().manual_seed(11)
    n, zero = 150, (0, 64, 149)
    L = torch.tril(torch.rand(n, n, generator=g, dtype=F64)) / n + torch.eye(n, dtype=F64)
    for j in zero:
        L[j, j] = 0
        L[j + 1:, j] = 0
    B = torch.randn(n, 9, generator=g, dtype=F64)
    for transpose in (False, True):
        got = lib.gp_trsm(L.cuda(), B.clone().cuda(), transpose=transpose).cpu()
        assert all(torch.all(got[j] == 0) for j in zero) and torch.isfinite(got).all()
        ref = R.tri_solve(L, B, transpose)
        assert torch.allclose(got, ref, rtol=0, atol=1e-12 * ref.abs().max())


def test_trsm_random_within_backward_error_bounds(lib):
    g = torch.Generator().manual_seed(12)
    for n, ncols in ((300, 77), (1000, 3)):
        L = torch.tril(torch.randn(n, n, generator=g, dtype=F64)) / math.sqrt(n) + 2 * torch.eye(n, dtype=F64)
        B = torch.randn(n, ncols, generator=g, dtype=F64)
        for transpose in (False, True):
            X = lib.gp_trsm(L.cuda(), B.clone().cuda(), transpose=transpose).cpu()
            Lo = L.T if transpose else L
            bound = 2 * n * U * (Lo.abs() @ X.abs())
            assert ((Lo @ X - B).abs() <= bound).all(), (n, transpose)


def test_trsm_column_subset_gives_the_same_bits(lib):
    g = torch.Generator().manual_seed(13)
    n = 333
    L = torch.tril(torch.randn(n, n, generator=g, dtype=F64)) / math.sqrt(n) + 2 * torch.eye(n, dtype=F64)
    B = torch.randn(n, 100, generator=g, dtype=F64)
    idx = torch.tensor([3, 4, 40, 41, 99])
    for transpose in (False, True):
        full = lib.gp_trsm(L.cuda(), B.clone().cuda(), transpose=transpose).cpu()
        part = lib.gp_trsm(L.cuda(), B[:, idx].contiguous().cuda(), transpose=transpose).cpu()
        assert same_bits(part, full[:, idx])


# ------------------------------------------------------------------------------------------------ the model
def cond(case):
    p = case["params"]
    tx = torch.cat([f[0] for f in case["fits"]]).double()
    A = R.SqExp(p["s"], p["ell"]).double()(tx, tx).detach()
    A += float(torch.tensor(case["noise"])) * torch.eye(len(tx), dtype=F64)
    return float(torch.linalg.cond(A)), len(tx)


def within(got, ref, rel, what, floor=0.0):
    got = got.detach().cpu().to(ref.dtype)
    scale = max(float(ref.abs().max()), floor)
    err = float((got.to(F64) - ref.to(F64)).abs().max())
    assert err <= rel * scale, f"{what}: |err| {err:.3e} > {rel:.3e} x {scale:.3e}"
    return err / (rel * scale) if rel * scale else 0.0


@pytest.mark.parametrize("name", ["notebook", "d3", "multi", "fp32"])
def test_model_matches_the_reference_fixture(lib, fixture, name):
    case = fixture[name]
    kappa, M = cond(case)
    steps, mu, sig, grads = R.replay(case, R.model_predict, device="cuda")
    fp32 = name == "fp32"
    u = 2.0 ** -24 if fp32 else U
    rel = 16 * M * kappa * u
    for (m, s), (fm, fs) in zip(steps, case["steps"]):
        assert m.dtype == fm.dtype and s.dtype == fs.dtype and m.shape == fm.shape and s.shape == fs.shape
        within(m, fm, rel, f"{name} mu")
        within(s, fs, rel, f"{name} sig")
    grel = 16 * M * kappa * kappa * u if not fp32 else 64 * kappa * u * M
    for k, ref in case["grads"].items():
        assert grads[k].dtype == ref.dtype and grads[k].shape == ref.shape, k
        within(grads[k], ref, min(grel, 0.05), f"{name} d{k}", floor=1.0 if ref.dim() == 0 else 0.0)


def _posterior_parts(M, N, D, g, dup=None, noise=0.0):
    tx = torch.rand(M, D, generator=g, dtype=F64) * 4
    if dup is not None:
        tx = torch.cat([tx, tx[dup:dup + 1]])
    ty = torch.sin(tx).sum(1, keepdim=True)
    x = torch.rand(N, D, generator=g, dtype=F64) * 4
    return tx, ty, x


def test_duplicate_point_is_conditioned_out_with_zero_gradients(lib):
    from pytorch_generative_b200.models import GaussianProcess

    g = torch.Generator().manual_seed(20)
    tx, ty, x = _posterior_parts(80, 33, 3, g, dup=17)
    mean, kernel = R.ConstMean(0.1).cuda(), R.SqExp(1.0, 0.6).cuda()
    gp = GaussianProcess(mean, kernel)
    txc, tyc, xc = tx.cuda().requires_grad_(True), ty.cuda().requires_grad_(True), x.cuda()
    gp.fit(txc, tyc)
    mu, sig = gp.predict(xc)
    assert int(gp.dropped) == 1
    ref = GaussianProcess(mean, kernel)
    ref.fit(tx[:80].cuda(), ty[:80].cuda())
    with torch.no_grad():
        rmu, rsig = ref.predict(xc)
    kappa, _ = cond(dict(params=dict(s=1.0, ell=0.6), fits=[(tx[:80], None)], noise=0.0))
    within(mu, rmu.cpu(), 64 * 80 * kappa * U, "mu")
    within(sig, rsig.cpu(), 64 * 80 * kappa * U, "sig")
    (mu.sum() + sig.sum()).backward()
    assert torch.all(txc.grad[80] == 0) and torch.all(tyc.grad[80] == 0)
    assert txc.grad[:80].abs().max() > 0


def test_rank_deficient_prior_grid_samples(lib):
    from pytorch_generative_b200.models import GaussianProcess

    gp = GaussianProcess(R.ConstMean(), R.SqExp())
    grid = torch.linspace(0, 6, 100, dtype=F64)[:, None].cuda()
    with pytest.raises(torch.linalg.LinAlgError):
        torch.linalg.cholesky(R.SqExp().double()(grid.cpu(), grid.cpu()).detach())
    torch.manual_seed(0)
    s = gp.sample(grid, 5)
    assert s.shape == (5, 100) and s.dtype == F64 and s.is_cuda and torch.isfinite(s).all()
    assert int(gp.dropped) > 0


def test_thompson_loop_on_the_device(lib):
    from pytorch_generative_b200.models import GaussianProcess

    torch.manual_seed(1)
    fn = lambda t: torch.sin(2 * t) + 0.3 * t
    grid = torch.linspace(0, 6, 100, dtype=F64)[:, None].cuda()
    gp = GaussianProcess(R.ConstMean().cuda(), R.SqExp().cuda(), 0.1 ** 2)
    for _ in range(8):
        s = gp.sample(grid, 1)
        assert s.is_cuda and torch.isfinite(s).all()
        x_next = grid[s[0].argmax()][None]
        gp.fit(x_next, fn(x_next) + 0.1 * torch.randn(1, 1, dtype=F64, device="cuda"))
    assert gp.train_x.shape == (8, 1)
    mu, sig = gp.predict(grid)
    assert torch.isfinite(mu).all() and torch.isfinite(sig).all()


def _fitted(M, N, D, seed, noise=1e-2):
    from pytorch_generative_b200.models import GaussianProcess

    g = torch.Generator().manual_seed(seed)
    tx, ty, x = _posterior_parts(M, N, D, g)
    gp = GaussianProcess(R.ConstMean(0.2).cuda(), R.SqExp(1.0, 0.8).cuda(), noise)
    gp.fit(tx.cuda(), ty.cuda())
    return gp, x.cuda()


def test_sample_is_mu_plus_z_lt(lib):
    gp, x = _fitted(100, 40, 2, 30)
    with torch.no_grad():
        mu, sig = gp.predict(x)
    torch.manual_seed(5)
    s = gp.sample(x, 7)
    torch.manual_seed(5)
    z = torch.randn(7, 40, dtype=F64, device="cuda")
    Ls, dropped = potrf(lib, sig.cpu())
    assert dropped == 0
    ref = mu.cpu().T + z.cpu() @ Ls.T
    bound = 40 * 2.0 ** -52 * (mu.cpu().abs().T + z.cpu().abs() @ Ls.abs().T)
    assert ((s.cpu() - ref).abs() <= bound).all()
    assert ((Ls @ Ls.T - sig.cpu()).abs() <= 2 * 40 * U * (Ls.abs() @ Ls.abs().T)).all()


def test_sample_statistics(lib):
    gp, x = _fitted(60, 32, 2, 31, noise=1e-1)
    with torch.no_grad():
        mu, sig = gp.predict(x)
    S = 200_000
    torch.manual_seed(6)
    s = gp.sample(x, S).cpu()
    mu, sig = mu.cpu().reshape(-1), sig.cpu()
    d = sig.diagonal()
    assert ((s.mean(0) - mu).abs() <= 5 * (d / S).sqrt() + 1e-12).all()
    c = s - mu
    emp = c.T @ c / S
    sd = ((d[:, None] * d[None, :] + sig ** 2) / S).sqrt()
    assert ((emp - sig).abs() <= 5 * sd + 1e-12).all()


def test_repeat_runs_and_sub_batches_are_bit_identical(lib):
    gp, x = _fitted(300, 90, 3, 32)
    with torch.no_grad():
        mu, sig = gp.predict(x)
        mu2, sig2 = gp.predict(x)
        idx = torch.tensor([0, 5, 6, 50, 89], device="cuda")
        smu, ssig = gp.predict(x[idx])
    assert same_bits(mu, mu2) and same_bits(sig, sig2)
    assert same_bits(smu, mu[idx]) and same_bits(ssig, sig[idx][:, idx])


@pytest.mark.parametrize("M", [1, 64, 65, 200])
def test_launch_count_formula(lib, M):
    gp, x = _fitted(M, 20, 2, 33)
    T = -(-M // NB)
    before = lib.launch_count()
    with torch.no_grad():
        gp.predict(x)
    assert lib.launch_count() - before == 5 * T - 1
    x = x.clone().requires_grad_(True)
    mu, sig = gp.predict(x)
    before = lib.launch_count()
    (mu.sum() + sig.sum()).backward()
    assert lib.launch_count() - before == 2 * T - 1 + 5


def test_predict_and_backward_under_cuda_graph_capture(lib):
    gp, x = _fitted(150, 40, 2, 34)
    gp.train_x.requires_grad_(True)
    xs = x.clone().requires_grad_(True)
    params = [xs, gp.train_x, *gp.mean.parameters(), *gp.kernel.parameters()]
    g = torch.Generator().manual_seed(35)
    c1 = torch.randn(40, 1, generator=g, dtype=F64).cuda()
    c2 = torch.randn(40, 40, generator=g, dtype=F64).cuda()

    def step():
        mu, sig = gp.predict(xs)
        return (mu, sig, *torch.autograd.grad((mu * c1).sum() + (sig * c2).sum(), params))

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = [t.detach().clone() for t in step()]
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, eager):
        assert same_bits(a.detach(), b)


def test_large_case_against_float64_cpu(lib):
    from pytorch_generative_b200.models import GaussianProcess

    g = torch.Generator().manual_seed(40)
    M, N, D = 8192, 2048, 8
    tx = torch.rand(M, D, generator=g, dtype=F64) * 6
    ty = torch.sin(tx).sum(1, keepdim=True)
    x = torch.rand(N, D, generator=g, dtype=F64) * 6
    noise = 1e-2
    mean, kernel = R.ConstMean(0.1), R.SqExp(1.0, 1.5)
    c1 = torch.randn(N, 1, generator=g, dtype=F64)
    c2 = torch.randn(N, N, generator=g, dtype=F64)

    def run(predict, dev):
        m, k = R.ConstMean(0.1).to(dev), R.SqExp(1.0, 1.5).to(dev)
        a, b, q = tx.to(dev).requires_grad_(True), ty.to(dev).requires_grad_(True), x.to(dev).requires_grad_(True)
        mu, sig = predict(m, k, a, b, q)
        ((mu * c1.to(dev)).sum() + (sig * c2.to(dev)).sum()).backward()
        return [t.detach().cpu() for t in (mu, sig, q.grad, a.grad, b.grad, k.s.grad, k.ell.grad, m.c.grad)]

    def ours(m, k, a, b, q):
        gp = GaussianProcess(m, k, noise)
        gp.fit(a, b)
        return gp.predict(q)

    def cpu(m, k, a, b, q):
        A = k(a, a) + float(torch.tensor(noise)) * torch.eye(M, dtype=F64)
        Lc = torch.linalg.cholesky(A)
        V = torch.linalg.solve_triangular(Lc, k(a, q), upper=False)
        beta = torch.linalg.solve_triangular(Lc, b - m(a), upper=False)
        return m(q) + V.T @ beta, k(q, q) - V.T @ V

    got = run(ours, "cuda")
    ref = run(cpu, "cpu")
    # kappa <= (max row sum of |K| + noise) / noise: Gershgorin above, the noise below
    kappa = (float(kernel(tx, tx).detach().abs().sum(1).max()) + noise) / noise
    names = ["mu", "sig", "dx", "dtrain_x", "dtrain_y", "ds", "dell", "dc"]
    for i, (a, b) in enumerate(zip(got, ref)):
        rel = 16 * M * kappa * U * (1 if i < 2 else kappa)
        within(a, b, min(rel, 1e-3), names[i], floor=1.0 if b.dim() == 0 else 0.0)
