"""Minimal stand-ins for the third-party modules the MER2024 VideoMAE package (feature_extraction/visual/videomae)
imports but this image lacks: timm's layers / registry / create_model / utils.get_state_dict, tensorboardX and
torch._six.  Only what that package calls, with timm's semantics; used by make_golden_sun_videomae.py."""
import math
import sys
import types

import torch

_REGISTRY = {}


def drop_path(x, drop_prob=0.0, training=False):
    if drop_prob == 0.0 or not training:
        return x
    keep = 1 - drop_prob
    mask = x.new_empty((x.shape[0],) + (1,) * (x.ndim - 1)).bernoulli_(keep)
    return x * mask / keep


def to_2tuple(x):
    return tuple(x) if isinstance(x, (list, tuple)) else (x, x)


def trunc_normal_(tensor, mean=0.0, std=1.0, a=-2.0, b=2.0):
    return torch.nn.init.trunc_normal_(tensor, mean, std, a, b)


def register_model(fn):
    _REGISTRY[fn.__name__] = fn
    return fn


def create_model(model_name, pretrained=False, **kwargs):
    """timm.create_model: kwargs whose value is None are dropped before the entry point is called."""
    kwargs = {k: v for k, v in kwargs.items() if v is not None}
    return _REGISTRY[model_name](pretrained=pretrained, **kwargs)


def get_state_dict(model, unwrap_fn=None):
    return model.state_dict()


class SummaryWriter:
    def __init__(self, *a, **k):
        pass


def install():
    """Register the stand-ins in sys.modules (idempotent)."""
    timm = types.ModuleType("timm")
    models = types.ModuleType("timm.models")
    layers = types.ModuleType("timm.models.layers")
    registry = types.ModuleType("timm.models.registry")
    utils = types.ModuleType("timm.utils")
    layers.drop_path, layers.to_2tuple, layers.trunc_normal_ = drop_path, to_2tuple, trunc_normal_
    registry.register_model = register_model
    models.create_model, models.layers, models.registry = create_model, layers, registry
    utils.get_state_dict = get_state_dict
    timm.models, timm.utils = models, utils
    tbx = types.ModuleType("tensorboardX")
    tbx.SummaryWriter = SummaryWriter
    six = types.ModuleType("torch._six")
    six.inf = math.inf
    sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers,
                        "timm.models.registry": registry, "timm.utils": utils, "tensorboardX": tbx,
                        "torch._six": six})
