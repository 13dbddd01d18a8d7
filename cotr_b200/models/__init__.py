"""Mirror of the reference's COTR/models package for the inference hot path.

`build_model(args)` (reference: COTR/models/__init__.py:9-10) returns an nn.Module with the reference's 381-entry
state_dict schema whose forward runs the hand-written sm_90a kernels through the C ABI.
"""
from .cotr_model import COTR, build


def build_model(args):
    return build(args)
