"""Eager MC steps of BBBAlexNet (B=512, LRT, fused chain + MC exchange kernel) for ncu captures:
    ncu --set full --import-source on -k regex:"conv_s4_kernel|tap_gemm_kernel|mc_exchange_kernel" -s 14 -c 7 -o prof python tools/ncu_mc.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_bayesiancnn_b200 import mc
from bench import build_net
dev = torch.device("cuda:0")
from pytorch_bayesiancnn_b200 import _lib as L
if os.environ.get("NCU_WIDE_TILES", "0") == "1":          # the tile policy of the in-flight engines (bbb_set_wide_tiles)
    L.lib().bbb_set_wide_tiles(1)
net = build_net(sys.argv[1] if len(sys.argv) > 1 else "lrt", 10, dev, "bf16")
xs = [torch.randn(512, 3, 32, 32, device=dev) for _ in range(4)]
eng = mc.MCForward(net, xs[0], 1, seed=1, graph=False)
for x in xs:
    out = eng(x)
torch.cuda.synchronize()
print("ok", float(out["kl"]))
