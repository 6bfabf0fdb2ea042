"""instantiate_from_config / get_obj_from_str: the YAML `target:` -> class lookup that is the reference's
plugin mechanism (model_lib/ControlNet/ldm/util.py:72-87), plus a dependency-free create_model
(model_lib/ControlNet/cldm/model.py:24-28; the reference needs omegaconf, PyYAML is enough here)."""
from __future__ import annotations

import importlib


class AttrDict(dict):
    """Plain-dict config node with attribute access (what the scripts use of OmegaConf: config.model)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def to_attr(o):
    if isinstance(o, dict):
        return AttrDict({k: to_attr(v) for k, v in o.items()})
    if isinstance(o, (list, tuple)):
        return [to_attr(v) for v in o]
    return o


def get_obj_from_str(string, reload=False):
    module, cls = string.rsplit(".", 1)
    mod = importlib.import_module(module)
    if reload:
        mod = importlib.reload(mod)
    return getattr(mod, cls)


def instantiate_from_config(config):
    if "target" not in config:
        if config in ("__is_first_stage__", "__is_unconditional__"):
            return None
        raise KeyError("Expected key `target` to instantiate.")
    return get_obj_from_str(config["target"])(**config.get("params", dict()))


def load_config(path):
    try:
        from omegaconf import OmegaConf  # used when available, like the reference
        return OmegaConf.load(path)
    except ImportError:
        import yaml
        with open(path) as f:
            return to_attr(yaml.safe_load(f))


def create_model(config_path):
    config = load_config(config_path)
    model = instantiate_from_config(config.model).cpu()
    print(f"Loaded model config from [{config_path}]")
    return model


def _one(lst):
    """a conditioning list as one tensor (torch.cat over channels).  A one-element list (every released script) is
    passed on as the caller's tensor: the engine caches per tensor identity, and a fresh copy would miss every call."""
    import torch
    return lst[0] if len(lst) == 1 else torch.cat(lst, 1)


def get_state_dict(container):
    """a checkpoint file holds either the parameter dict itself or {'state_dict': parameter dict, ...}"""
    inner = container.get("state_dict") if isinstance(container, dict) else None
    return container if inner is None else inner


def load_state_dict(ckpt_path, location="cpu"):
    """name -> tensor of a .ckpt/.pth (torch pickle) or .safetensors checkpoint, tensors placed on `location`
    (the signature of the reference's cldm/model.py:12-21; the released MagicPose weights are a .pth)"""
    import torch
    if str(ckpt_path).lower().endswith(".safetensors"):
        from safetensors.torch import load_file
        tensors = load_file(ckpt_path, device=location)
    else:
        tensors = torch.load(ckpt_path, map_location=torch.device(location))
    tensors = get_state_dict(tensors)
    print(f"Loaded state_dict from [{ckpt_path}]")
    return tensors
