"""The LRT activation noise the fused tensor-core chain draws in-kernel (Philox, element index = NHWC-flat index of the
pre-pool output) must be exactly the stream bbb_philox_normal_fill draws: the chain run on its own noise and the same
chain fed that stream as external eps give bit-identical logits.  The tap-GEMM producer warps draw the noise of a tile
while its main loop runs, so this covers their (row, pixel, channel) -> element mapping for both tile widths, pooled and
unpooled layers, the classifier's N % 4 != 0 fallback and a ragged last row tile."""
import pytest
import torch

from tests.test_gpu_mc import _engine_eps, _net

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


@pytest.mark.parametrize("batch, wide", [(512, False), (512, True), (200, False), (200, True)])
def test_fused_lrt_noise_equals_external_draw(dev, batch, wide):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import _lib as L
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "bf16")
    with torch.no_grad():                              # sigma ~ 0.13: the noise term is far above bf16 rounding
        for name, p in net.named_parameters():
            if name.endswith("_rho"):
                p.fill_(-2.0)
    x = torch.randn(batch, 3, 32, 32, generator=torch.Generator().manual_seed(5)).to(dev)
    seed, stream0 = 31, 500
    prev = L.lib().bbb_set_wide_tiles(1 if wide else 0)
    try:
        bbb.manual_seed(seed, stream0)
        with torch.no_grad():
            a, kl_a = net(x)
        eps = _engine_eps(bbb, "alexnet", 10, 3, "lrt", batch, seed, stream0, dev)
        with torch.no_grad(), bbb.external_eps(eps):
            b, kl_b = net(x)
        torch.cuda.synchronize()
    finally:
        L.lib().bbb_set_wide_tiles(prev)
    assert net._fused_plans.get((batch, 3, 32, 32)) is not None, "the fused tensor-core chain did not run"
    assert torch.isfinite(a).all()
    assert torch.equal(a, b), float((a - b).abs().max())
    assert float(kl_a) == float(kl_b)
