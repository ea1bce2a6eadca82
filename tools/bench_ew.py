"""GB/s of the BatchNorm row kernels at the shapes of the training step (tuning aid).  The rows-in-flight factors are
developer knobs read once per process from the environment (csrc/elementwise.cu: PNX_BN_BWD_APPLY_U,
PNX_BN_BWD_REDUCE_U, PNX_BN_BWD_REDUCE_WAVES, PNX_BN_BWD_APPLY_WAVES); run once per setting."""
import os, sys, torch
sys.path.insert(0, '.')
from pillarnext_b200 import ops

def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

dev = 'cuda'
print("env:", {k: v for k, v in os.environ.items() if k.startswith("PNX_")})
tot = {"apply": 0.0, "reduce": 0.0, "bwd_apply": 0.0}
# (M, C, launches per step) of the nuScenes training step
for (M, C, n) in [(677376, 384, 6), (169344, 256, 14), (677376, 64, 6), (140000, 64, 5), (60000, 128, 4), (25000, 256, 4)]:
    x = torch.randn(M, C, device=dev).bfloat16()
    dy = torch.randn(M, C, device=dev).bfloat16()
    y = torch.empty_like(x); dx = torch.empty_like(x)
    sc = torch.rand(C, device=dev) + 0.5; sh = torch.randn(C, device=dev)
    mean = torch.randn(C, device=dev) * 0.1; invstd = torch.rand(C, device=dev) + 0.5
    gamma = torch.ones(C, device=dev)
    red = torch.zeros(2 * C, dtype=torch.float64, device=dev)
    t_apply = timeit(lambda: ops.bn_apply(x, M, C, sc, sh, y, relu=True))
    def reduce_only():
        ops.bn_bwd_reduce(dy, None, x, M, C, mean, invstd, True, (sc, sh), red=red)
    def apply_only():   # the apply after a reduce fused into the GEMM epilogue: dy is the gated g, no mask
        ops.bn_bwd_apply(dy, None, x, M, C, mean, invstd, gamma, red, M, False, (sc, sh), dx)
    def apply_mask():   # the un-fused apply: recomputed ReLU mask
        ops.bn_bwd_apply(dy, None, x, M, C, mean, invstd, gamma, red, M, True, (sc, sh), dx)
    t_red, t_app, t_appm = timeit(reduce_only), timeit(apply_only), timeit(apply_mask)
    b = M * C * 2
    tot["apply"] += n * t_apply; tot["reduce"] += n * t_red; tot["bwd_apply"] += n * t_appm
    print(f"M={M} C={C}: bn_apply {t_apply*1e3:.0f} us {2*b/t_apply/1e6:.0f} GB/s | reduce {t_red*1e3:.0f} us {2*b/t_red/1e6:.0f} GB/s"
          f" | bwd apply (no mask) {t_app*1e3:.0f} us {3*b/t_app/1e6:.0f} GB/s | bwd apply (mask) {t_appm*1e3:.0f} us {3*b/t_appm/1e6:.0f} GB/s")
print("step estimate (ms):", {k: round(v, 3) for k, v in tot.items()})
