"""Record how the original project's UNMODIFIED model files assemble on this repository's `layers` package.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_dropin.py /path/to/PyTorch-BayesianCNN

Imports models/BayesianModels/*.py from the original project with this repository's `layers` resolving first
and writes, per (model, layer type), the state_dict keys and shapes and the child module types to dropin.json
next to this script.  tests/test_dropin.py checks this repository's own model classes against that record, so
the suite needs no copy of the original project.
"""
import importlib
import json
import os
import sys

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CFG_PRIORS = {"prior_mu": 0, "prior_sigma": 0.1,
              "posterior_mu_initial": (0, 0.1), "posterior_rho_initial": (-5, 0.1)}
MODELS = (("alexnet", "BayesianAlexNet", "BBBAlexNet", 3), ("lenet", "BayesianLeNet", "BBBLeNet", 3),
          ("3conv3fc", "Bayesian3Conv3FC", "BBB3Conv3FC", 1))


def main(ref):
    sys.path[:] = [ROOT] + [p for p in sys.path if p not in (ROOT, ref)] + [ref]
    import layers
    assert os.path.dirname(os.path.abspath(layers.__file__)) == os.path.join(ROOT, "layers")
    out = {}
    for key, mod, cls, cin in MODELS:
        m = importlib.import_module(f"models.BayesianModels.{mod}")
        assert m.__file__.startswith(os.path.abspath(ref))
        for lt in ("lrt", "bbb"):
            net = getattr(m, cls)(10, cin, CFG_PRIORS, lt, "softplus")
            out[f"{key}/{lt}"] = {"cls": cls, "inputs": cin,
                                  "state_dict": [[k, list(v.shape)] for k, v in net.state_dict().items()],
                                  "children": [type(c).__name__ for c in net.children()]}
        try:
            getattr(m, cls)(10, cin, CFG_PRIORS, "nope")
            raise AssertionError("the original model accepted an unknown layer type")
        except ValueError:
            pass
    with open(os.path.join(HERE, "dropin.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
