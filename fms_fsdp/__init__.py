"""Compatibility alias: ``fms_fsdp.*`` resolves to the H100-native implementation ``fms_fsdp_b200.*`` so
code written against the reference's public API (``from fms_fsdp.config import train_config``,
``from fms_fsdp.policies import ...``, ``from fms_fsdp.utils.train_utils import train`` ...) runs unchanged."""
import importlib
import sys

import fms_fsdp_b200 as _impl

_SUBMODULES = [
    "config", "config.training", "policies", "policies.ac_handler", "policies.mixed_precision",
    "policies.param_init", "policies.wrapping", "utils", "utils.config_utils", "utils.train_utils",
    "utils.checkpointing_utils", "utils.dataloader_utils", "utils.dataset_utils", "models", "parallel", "ops",
]


def _alias():
    for name in _SUBMODULES:
        try:
            mod = importlib.import_module(f"fms_fsdp_b200.{name}")
        except ImportError:
            continue
        sys.modules[f"fms_fsdp.{name}"] = mod
        parent, _, leaf = name.rpartition(".")
        if not parent:
            globals()[leaf] = mod


_alias()
__version__ = getattr(_impl, "__version__", "0.1.0")
