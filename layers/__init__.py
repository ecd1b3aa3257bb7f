"""Drop-in replacement for the reference's top-level ``layers`` package
(layers/__init__.py:1-7): same six names, backed by the H100 engine."""
from pytorch_bayesiancnn_b200 import (BBB_Linear, BBB_Conv2d, BBB_LRT_Linear, BBB_LRT_Conv2d,
                                      FlattenLayer, ModuleWrapper)
