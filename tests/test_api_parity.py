"""Every public top-level name (and public method) of the original project's modules must exist under the same import
path (`fms_fsdp.*` aliases to `fms_fsdp_b200.*`).  The original names and parameter lists are recorded in
tests/golden/reference_api.json.gz (oracle/make_golden.py)."""
import gzip
import importlib
import json
import os

import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_api.json.gz")
MODULES = {
    "fms_fsdp/config/training.py": "fms_fsdp.config.training",
    "fms_fsdp/utils/config_utils.py": "fms_fsdp.utils.config_utils",
    "fms_fsdp/utils/train_utils.py": "fms_fsdp.utils.train_utils",
    "fms_fsdp/utils/checkpointing_utils.py": "fms_fsdp.utils.checkpointing_utils",
    "fms_fsdp/utils/dataloader_utils.py": "fms_fsdp.utils.dataloader_utils",
    "fms_fsdp/utils/dataset_utils.py": "fms_fsdp.utils.dataset_utils",
    "fms_fsdp/policies/ac_handler.py": "fms_fsdp.policies.ac_handler",
    "fms_fsdp/policies/mixed_precision.py": "fms_fsdp.policies.mixed_precision",
    "fms_fsdp/policies/wrapping.py": "fms_fsdp.policies.wrapping",
    "fms_fsdp/policies/param_init.py": "fms_fsdp.policies.param_init",
    "speculator/train_speculator_utils.py": "speculator.train_speculator_utils",
    "speculator/train_speculator.py": "speculator.train_speculator",
    "fms_to_hf_llama.py": "fms_to_hf_llama",
    "fms_to_hf_mamba.py": "fms_to_hf_mamba",
    "main_training_llama.py": "main_training_llama",
    "main_training_mamba.py": "main_training_mamba",
}


def _recorded(path):
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)[path]


@pytest.mark.parametrize("path,mod", sorted(MODULES.items()))
def test_public_names_of_reference_module_exist(path, mod):
    rec = _recorded(path)
    ours = importlib.import_module(mod)
    missing = [n for n in rec["names"] if not hasattr(ours, n)]
    for cname, methods in rec["classes"].items():
        if cname.startswith("_") or not hasattr(ours, cname):
            continue
        cls = getattr(ours, cname)
        missing += [f"{cname}.{m}" for m in methods if not m.startswith("_") and not hasattr(cls, m)]
    assert not missing, f"{mod} lacks {missing}"


def _positional_names(fn_node):
    a = fn_node.args
    return [x.arg for x in a.posonlyargs + a.args if x.arg not in ("self", "cls")], [x.arg for x in a.kwonlyargs]


@pytest.mark.parametrize("path,mod", sorted(MODULES.items()))
def test_signatures_accept_the_reference_call_forms(path, mod):
    """Every public function / method (and ``__init__``) takes the reference's parameters under the same names and, unless it
    takes ``*args``, at the same positions -- so both keyword and positional call sites of reference users keep working."""
    import inspect
    rec = _recorded(path)
    ours = importlib.import_module(mod)
    problems = []

    def check(recorded, obj, label):
        try:
            params = list(inspect.signature(obj).parameters.values())
        except (TypeError, ValueError):
            return
        names = [p.name for p in params if p.name not in ("self", "cls")]
        var_kw = any(p.kind == p.VAR_KEYWORD for p in params)
        var_pos = any(p.kind == p.VAR_POSITIONAL for p in params)
        pos, kwonly = recorded
        for i, n in enumerate(pos):
            if n not in names:
                if not var_kw:
                    problems.append(f"{label}: no parameter {n}")
            elif names.index(n) != i and not var_pos:
                problems.append(f"{label}: {n} is parameter {names.index(n)}, reference has it at {i}")
        problems.extend(f"{label}: no keyword {n}" for n in kwonly if n not in names and not var_kw)

    for name, sig in rec["functions"].items():
        if hasattr(ours, name):
            check(sig, getattr(ours, name), name)
    for cname, methods in rec["classes"].items():
        if hasattr(ours, cname):
            cls = getattr(ours, cname)
            for m, sig in methods.items():
                if hasattr(cls, m):
                    check(sig, getattr(cls, m), f"{cname}.{m}")
    assert not problems, f"{mod}: {problems}"
