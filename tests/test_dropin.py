"""The original project's model files on top of this repo's `layers` package.

tests/golden/dropin.json records what models/BayesianModels/*.py of the original project build when this
repository's `layers` resolves first (tests/golden/make_dropin.py): state_dict keys and shapes and child module
types.  Our own model classes must build the same, so checkpoints are interchangeable and the original model
files run unchanged on the engine."""
import json
import os

import pytest
import torch

from tests.conftest import GOLDEN
from tests.util import CFG_PRIORS


@pytest.fixture(scope="module")
def dropin():
    with open(os.path.join(GOLDEN, "dropin.json")) as f:
        return json.load(f)


def test_reference_model_files_build_on_our_layers(dropin):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import models as ours
    assert sorted(dropin) == sorted(f"{m}/{lt}" for m in ("alexnet", "lenet", "3conv3fc") for lt in ("lrt", "bbb"))
    for key, rec in dropin.items():
        lt = key.split("/")[1]
        our_cls = getattr(ours, rec["cls"])
        mine = our_cls(10, rec["inputs"], CFG_PRIORS, lt, "softplus")
        assert isinstance(mine, bbb.ModuleWrapper)
        assert [[k, list(v.shape)] for k, v in mine.state_dict().items()] == rec["state_dict"], key
        assert [type(m).__name__ for m in mine.children()] == rec["children"], key
        state = {k: torch.randn(shape) for k, shape in rec["state_dict"]}
        mine.load_state_dict(state)                                      # checkpoints are interchangeable
        with pytest.raises(ValueError):
            our_cls(10, rec["inputs"], CFG_PRIORS, "nope")


@pytest.mark.gpu
def test_reference_model_files_run_on_the_engine(dropin):
    """Runs this package's restated BBBLeNet (models.py), not the original model file: the stored record ties the two
    together (same state_dict layout), and the run checks that a ReLU BBB net goes through the engine end to end."""
    from pytorch_bayesiancnn_b200 import models as ours
    rec = dropin["lenet/bbb"]
    net = getattr(ours, rec["cls"])(10, 3, CFG_PRIORS, "bbb", "relu").cuda().train()
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == rec["state_dict"]
    with torch.no_grad():
        out, kl = net(torch.randn(5, 3, 32, 32, device="cuda"))
    assert out.shape == (5, 10) and kl.dim() == 0 and torch.isfinite(out).all()
