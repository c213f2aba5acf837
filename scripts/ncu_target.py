"""Short launch sequences for `ncu --set full` captures (one GPU).

    ncu --set full --clock-control none --import-source on -k regex:gemm3_wgmma -s 3 -c 1 -o /tmp/pair python scripts/ncu_target.py gemm
    ncu --set full --clock-control none --import-source on -k regex:gae_tma -s 2 -c 1 -o /tmp/gae python scripts/ncu_target.py gae
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.networks import fused  # noqa: E402


def gemm():
    M, K = 16384, 256
    a = torch.randn(M, K, device="cuda")
    w = torch.randn(256, K, device="cuda") / 16
    bias = torch.randn(256, device="cuda") * 0.1
    pl = fused.split_tf32(w)
    g = torch.randn(M, 256, device="cuda")
    ws = torch.empty(64 * 256 * 256, device="cuda")
    for _ in range(6):
        ops.gemm3_pair(a, w, planes=pl, bias=bias, act=1)          # forward
    for _ in range(3):
        ops.gemm3_pair(g, w, planes=pl, b_nmajor=True)             # dgrad
    for _ in range(3):
        ops.gemm3_pair_tn(g, a, splits=64, workspace=ws)           # wgrad
    torch.cuda.synchronize()


def gae():
    T, N = 128, 1 << 20
    R = torch.randn(T, N, device="cuda")
    V = torch.randn(T, N, device="cuda")
    Tm = (torch.rand(T, N, device="cuda") < 0.01).to(torch.uint8)
    TL = (torch.rand(T, N, device="cuda") < 0.005).to(torch.uint8)
    LV = torch.randn(N, device="cuda")
    A, Rt = torch.empty_like(R), torch.empty_like(R)
    for variant in (4, 4, 4, 2, 2, 2):
        ops.gae_scan(R, V, Tm, TL, LV, 0.99, 0.95, True, A, Rt, variant)
    torch.cuda.synchronize()


if __name__ == "__main__":
    {"gemm": gemm, "gae": gae}[sys.argv[1]]()
