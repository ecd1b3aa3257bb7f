"""math='tf32': the tensor-core layer kernel with tf32 operands (fp32 storage rounded to a 10-bit mantissa, fp32
accumulators) -- what the reference's own GPU conv computes by default (SURVEY D9) -- against the oracle and the
reference-generated golden fixtures.  Bar: 1e-3 of the output scale per layer (north_star's fp32 bar), KL 1e-5."""
import pytest
import torch

from tests.util import CFG_PRIORS, build_layer_from_case, case_names, load_case, load_params_into, scale_err
from tests.test_gpu_parity import _grad_case, _lrt_eps_like, dev  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
TF32_TOL = 1e-3
KL_TOL = 1e-5


def test_tf32_layer_cases_external_eps(golden_layers, dev):
    import pytorch_bayesiancnn_b200 as bbb
    worst = 0.0
    for name in case_names(golden_layers):
        c = load_case(golden_layers, name)
        layer = build_layer_from_case(name, c, dev).train()
        layer.set_flag("math", "tf32")
        eps = [c["eps_w"]] + ([c["eps_b"]] if "eps_b" in c else []) if "_bbb_" in name else [c["eps_y"]]
        with torch.no_grad(), bbb.external_eps(eps):
            y = layer(c["x"].to(dev))
            kl = layer.kl_loss()
        e = scale_err(y, c["y"])
        worst = max(worst, e)
        assert e < TF32_TOL, (name, e)
        assert abs(float(kl) - float(c["kl"])) <= KL_TOL * abs(float(c["kl"])), (name, float(kl), float(c["kl"]))
        layer.eval()
        with torch.no_grad():
            ym = layer(c["x"].to(dev), sample=False)
        assert scale_err(ym, c["y_mean"]) < TF32_TOL, name
    print("tf32 layer cases worst scale err", worst)


def test_tf32_alexnet_layer_shapes_b512(dev):
    """Every BBBAlexNet layer geometry at the BASELINE batch (512), both variants, tf32 operands, identical eps."""
    import pytorch_bayesiancnn_b200 as bbb
    from oracle import bbb_oracle as O
    geoms = [(3, 64, 11, 4, 5, 32), (64, 192, 5, 1, 2, 4), (192, 384, 3, 1, 1, 2), (384, 256, 3, 1, 1, 2),
             (256, 128, 3, 1, 1, 2)]
    g = torch.Generator().manual_seed(11)
    worst = 0.0
    for variant, cls in (("bbb", bbb.BBB_Conv2d), ("lrt", bbb.BBB_LRT_Conv2d)):
        for (cin, cout, k, s, p, hw) in geoms:
            torch.manual_seed(cin)
            layer = cls(cin, cout, k, stride=s, padding=p, priors=CFG_PRIORS).to(dev).train()
            layer.set_flag("math", "tf32")
            x = torch.rand(512, cin, hw, hw, generator=g) * 2
            P = [t.detach().cpu() for t in (layer.W_mu, layer.W_rho, layer.bias_mu, layer.bias_rho)]
            ho = (hw + 2 * p - k) // s + 1
            if variant == "bbb":
                eps = [torch.randn(P[0].shape, generator=g), torch.randn(cout, generator=g)]
                ref = O.bbb_forward(x, *P, eps[0], eps[1], (s, p, 1))
            else:
                eps = [torch.randn(512, cout, ho, ho, generator=g)]
                ref = O.lrt_forward(x, *P, eps[0], (s, p, 1))
            with torch.no_grad(), bbb.external_eps(eps):
                y = layer(x.to(dev))
                kl = float(layer.kl_loss())
            e = scale_err(y, ref)
            worst = max(worst, e)
            refkl = float(O.kl_loss(*P, 0.0, 0.1))
            assert e < TF32_TOL, (variant, cin, cout, e)
            assert abs(kl - refkl) <= KL_TOL * abs(refkl)
    print("tf32 AlexNet layer shapes worst scale err", worst)


def test_tf32_model_cases_external_eps(golden_models, dev):
    """Whole models layer by layer on tf32 operands: 1e-3 on the logits of the whole model too (measured 4.3-6.7e-4; bf16
    chains measure 4-8e-3 on the same cases)."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import models as M
    from oracle import bbb_oracle as O
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}
    for name in case_names(golden_models):
        c = load_case(golden_models, name)
        key, inputs, outputs, variant, act, batch = [str(v) for v in c["meta"]]
        inputs, outputs, batch = int(inputs), int(outputs), int(batch)
        params = O.init_params(key, outputs, inputs, CFG_PRIORS, seed=123)
        net = load_params_into(cls[key](outputs, inputs, CFG_PRIORS, variant, act), params).to(dev).train()
        net.set_flag("math", "tf32")
        eps = O.draw_eps_like_reference(O.eps_shapes(key, outputs, inputs, variant, batch), seed=7)
        with torch.no_grad(), bbb.external_eps(eps):
            logits, kl = net(c["x"].to(dev))
        e = scale_err(logits, c["logits"])
        print(name, "tf32 whole-model scale err", e)
        assert e < TF32_TOL, (name, e)
        assert abs(float(kl) - float(c["kl"])) <= KL_TOL * abs(float(c["kl"])), (name, float(kl), float(c["kl"]))


def test_tf32_philox_equals_external_draw(dev):
    import pytorch_bayesiancnn_b200 as bbb
    for cls in (bbb.BBB_Conv2d, bbb.BBB_LRT_Conv2d):
        torch.manual_seed(4)
        layer = cls(16, 96, 3, padding=1, priors=CFG_PRIORS).to(dev).train()
        layer.set_flag("math", "tf32")
        x = torch.randn(40, 16, 6, 6, device=dev)
        bbb.manual_seed(77, 5)
        with torch.no_grad():
            y1 = layer(x)
        if cls is bbb.BBB_Conv2d:
            nw = layer.W_mu.numel()
            eps = [bbb.philox_normal(nw, 77, 5, 0, device=dev).view_as(layer.W_mu),
                   bbb.philox_normal(96, 77, 5, nw, device=dev)]
        else:
            eps = [_lrt_eps_like(bbb, y1, 77, 5, dev)]
        with torch.no_grad(), bbb.external_eps(eps):
            y2 = layer(x)
        assert scale_err(y1, y2) < 1e-6


def test_tf32_backward_matches_oracle_autograd(dev):
    """math='tf32': forward and the backward contractions (wgrad / dgrad as role-swapped calls of the layer kernel) on
    tf32 operands against torch autograd through the oracle."""
    for variant in ("bbb", "lrt"):
        for conv in (True, False):
            for bias in (True, False):
                _grad_case(dev, variant, conv, bias, True, math="tf32", tol_y=1e-3, tol_g=3e-3)
