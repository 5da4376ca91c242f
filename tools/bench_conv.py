"""Tap-loop convolution GEMMs (pg_gemm_bf16_conv) at the C3 / C4 layer shapes: fwd / dgrad / wgrad time and TFLOP/s,
next to the plain GEMM of the same M, N, K (what the tensor pipe would do without the shifted TMA boxes).
`python tools/bench_conv.py large` times a 7x7 CausalConv2d at 256 channels and a 256-channel PixelCNN step."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import _lib as L, ops
from pytorch_generative_b200.nn.tapconv import conv_taps

dev = torch.device("cuda:0")
BF16, F32 = torch.bfloat16, torch.float32
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=10):
    fn(); torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps


def case(label, n, h, w, cin, cout, kh, kw, pad):
    taps = conv_taps(kh, kw, pad[0], pad[1])
    T, P = len(taps), n * h * w
    x = torch.randn(P, cin, device=dev).to(BF16)
    dy = torch.randn(P, cout, device=dev).to(BF16)
    wcat = (torch.randn(cout, T * cin, device=dev) * 0.05).to(BF16)
    bias = torch.zeros(cout, device=dev)
    dw = torch.zeros(cout, T * cin, dtype=F32, device=dev)
    gf = 2.0 * P * cout * T * cin / 1e9
    if T == 1:
        rows = [("fwd", lambda: ops.linear_fwd(x, wcat, bias)), ("dgrad", lambda: ops.linear_dgrad(dy, wcat)),
                ("wgrad", lambda: ops.linear_wgrad(dy, x, dw))]
    else:
        rows = [("fwd", lambda: ops.conv_fwd(x, wcat, bias, n, h, w, taps)),
                ("dgrad", lambda: ops.conv_dgrad(dy, wcat, cin, n, h, w, taps)),
                ("wgrad", lambda: ops.conv_wgrad(dy, x, dw, n, h, w, taps))]
        xk = torch.randn(P, T * cin, device=dev).to(BF16)
        rows.append(("plain GEMM M=P N=cout K=T*cin", lambda: ops.linear_fwd(xk, wcat, bias)))
    for name, fn in rows:
        ms = timeit(fn)
        print(f"{label:34s} {name:30s} {ms * 1e3:8.1f} us  {gf / ms:8.1f} TFLOP/s", flush=True)


def variants_c4():
    """The epilogue variants the PixelSNAIL stack actually launches (nn/pm.py), at C4's shapes."""
    n, h, w, C = 128, 32, 32, 256
    P = n * h * w
    taps = conv_taps(2, 2, 1, 1)
    xa = torch.randn(P, C, device=dev).to(BF16)
    t = torch.randn(P, C, device=dev).to(BF16)
    w1 = (torch.randn(C, 4 * C, device=dev) * 0.05).to(BF16)
    w2 = (torch.randn(2 * C, 4 * C, device=dev) * 0.05).to(BF16)
    w11 = (torch.randn(C, C, device=dev) * 0.05).to(BF16)
    b1, b2 = torch.zeros(C, device=dev), torch.zeros(2 * C, device=dev)
    dy1 = torch.randn(P, C, device=dev).to(BF16)
    dy2 = torch.randn(P, 2 * C, device=dev).to(BF16)
    res = torch.randn(P, C, device=dev)
    gf1, gf2, gf11 = 2.0 * P * C * 4 * C / 1e9, 2.0 * P * 2 * C * 4 * C / 1e9, 2.0 * P * C * C / 1e9
    rows = [
        ("2x2 conv1 fwd: elu out only", gf1, lambda: ops.conv_fwd(xa, w1, b1, n, h, w, taps, act=L.ACT_ELU)),
        ("2x2 conv2 fwd: bf16 [P,512]", gf2, lambda: ops.conv_fwd(t, w2, b2, n, h, w, taps)),
        ("2x2 conv2 dgrad: elu' from out, bf16", gf2, lambda: ops.conv_dgrad(dy2, w2, C, n, h, w, taps, aux=t, dact=L.ACT_ELU_OUT)),
        ("2x2 conv1 dgrad: elu' from out, f32", gf1, lambda: ops.conv_dgrad(dy1, w1, C, n, h, w, taps, aux=xa, dact=L.ACT_ELU_OUT,
                                                                       want_f32=True, want_bf16=False)),
        ("2x2 conv1 dgrad: plain bf16", gf1, lambda: ops.conv_dgrad(dy1, w1, C, n, h, w, taps)),
        ("1x1 fwd: elu out only", gf11, lambda: ops.linear_fwd(xa, w11, b1, act=L.ACT_ELU)),
        ("1x1 fwd: f32 + res", gf11, lambda: ops.linear_fwd(xa, w11, b1, res0=res, want_bf16=False, want_f32=True)),
        ("1x1 dgrad: elu' from out, f32", gf11, lambda: ops.linear_dgrad(dy1, w11, aux=xa, dact=L.ACT_ELU_OUT, want_f32=True)),
        ("1x1 dgrad: elu' from out, bf16", gf11, lambda: ops.linear_dgrad(dy1, w11, aux=xa, dact=L.ACT_ELU_OUT)),
        ("1x1 dgrad: plain bf16", gf11, lambda: ops.linear_dgrad(dy1, w11)),
    ]
    for name, gf, fn in rows:
        ms = timeit(fn)
        print(f"c4 variant  {name:40s} {ms * 1e3:8.1f} us  {gf / ms:8.1f} TFLOP/s", flush=True)


def large():
    """A 7x7 mask-A CausalConv2d 256 -> 256 on 32x32 images, batch 64, forward + backward: the module (which takes the
    TMA tap loop here), and the 49-tap contraction at the ops level on the tap loop and on the gather path (tap gather,
    GEMM, tap scatter).  Then a PixelCNN(3, 3, 15, 256, 32) training step at batch 16, whose 7x7 input layer is too
    wide for the direct fp32 kernel."""
    from pytorch_generative_b200 import losses, models, nn, optim

    n, h, w, C, k = 64, 32, 32, 256, 7
    P = n * h * w
    taps = conv_taps(k, k, k // 2, k // 2)
    T = len(taps)
    gf = 3 * 2.0 * P * C * T * C / 1e9  # forward, dgrad and wgrad of the dense 49-tap contraction
    m = nn.CausalConv2d(True, C, C, k, padding=k // 2).to(dev)
    xm = torch.randn(n, C, h, w, device=dev, requires_grad=True)
    gm = torch.randn(n, C, h, w, device=dev)

    def module_step():
        m.weight.grad = m.bias.grad = xm.grad = None
        m(xm).backward(gm)

    x = torch.randn(P, C, device=dev).to(BF16)
    dy = torch.randn(P, C, device=dev).to(BF16)
    wcat = (torch.randn(C, T * C, device=dev) * 0.02).to(BF16)
    bias = torch.zeros(C, device=dev)
    dw = torch.zeros(C, T * C, dtype=F32, device=dev)
    xcat = torch.empty(P, T * C, dtype=BF16, device=dev)
    dx = torch.empty(P, C, dtype=BF16, device=dev)

    def tap_loop():
        ops.conv_fwd(x, wcat, bias, n, h, w, taps)
        ops.conv_dgrad(dy, wcat, C, n, h, w, taps)
        ops.conv_wgrad(dy, x, dw, n, h, w, taps)

    def gather():
        L.tap_gather(x, n, h, w, C, taps, L.ACT_NONE, xcat)
        ops.linear_fwd(xcat, wcat, bias)
        L.tap_scatter(ops.linear_dgrad(dy, wcat), n, h, w, C, taps, L.ACT_NONE, None, dx_bf16=dx)
        ops.linear_wgrad(dy, xcat, dw)

    for name, fn in [("CausalConv2d module fwd+bwd", module_step), ("tap loop fwd+dgrad+wgrad", tap_loop),
                     ("gather path fwd+dgrad+wgrad", gather)]:
        ms = timeit(fn)
        print(f"7x7A 256->256 (n=64, 32x32)  {name:30s} {ms * 1e3:9.1f} us  {gf / ms:8.1f} TFLOP/s", flush=True)

    torch.manual_seed(0)
    model = models.PixelCNN(3, 3, 15, 256, 32).to(dev)
    opt = optim.FusedAdam(model.parameters(), lr=1e-3)
    xb = torch.rand(16, 3, 32, 32, device=dev)

    def train_step():
        opt.zero_grad()
        losses.bce_with_logits_sum_mean(model(xb), xb).backward()
        opt.step()

    ms = timeit(train_step)
    print(f"PixelCNN(3, 3, 15, 256, 32) training step, batch 16, 32x32: {ms:.2f} ms  {16e3 / ms:.0f} images/s", flush=True)


which = sys.argv[1:] or ["c3", "c4"]
if "large" in which:
    large()
if "v4" in which:
    variants_c4()
if "c4" in which:
    case("c4 2x2 256->256 (n=128, 32x32)", 128, 32, 32, 256, 256, 2, 2, (1, 1))
    case("c4 2x2 256->512", 128, 32, 32, 256, 512, 2, 2, (1, 1))
    case("c4 1x1 256->256", 128, 32, 32, 256, 256, 1, 1, (0, 0))
if "c3" in which:
    case("c3 1x3 128->128 (n=128, 32x32)", 128, 32, 32, 128, 128, 1, 3, (0, 1))
    case("c3 2x1 128->256", 128, 32, 32, 128, 256, 2, 1, (2, 0))
    case("c3 1x2 128->256", 128, 32, 32, 128, 256, 1, 2, (0, 1))
    case("c3 1x1 256->256", 128, 32, 32, 256, 256, 1, 1, (0, 0))
    case("c3 1x1 128->128", 128, 32, 32, 128, 128, 1, 1, (0, 0))
