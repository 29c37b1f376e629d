"""Selective-recompute placement must reproduce the reference patterns bit-for-bit
(reference tests/test_selective_ac.py:12-64, rule at fms_fsdp/policies/ac_handler.py:43-58)."""
import pytest

from fms_fsdp_b200.models.llama import LLaMABlock
from fms_fsdp_b200.policies import apply_fsdp_checkpointing, is_checkpointed, selection_mask
from fms_fsdp_b200.policies.ac_handler import parse_fraction

T, F = True, False
CASES = [
    (0, [F] * 15), (1 / 100, [F] * 15), (-1, [F] * 15),
    (1 / 5, [F, F, T, F, F] * 3), (1 / 3, [F, T, F] * 5), (1 / 2, [T, F] * 7 + [T]),
    (3 / 5, [T, F, T, F, T] * 3), (2 / 3, [T, F, T] * 5), (1, [T] * 15), (5 / 3, [T] * 15),
    ("1/3", [F, T, F] * 5), ("1/2", [T, F] * 7 + [T]),
]


@pytest.mark.parametrize("p,expected", CASES)
def test_patterns(narrow_model_factory, p, expected):
    model = narrow_model_factory(15)
    apply_fsdp_checkpointing(model, LLaMABlock, p)
    assert [is_checkpointed(b) for b in model.layers] == expected
    assert selection_mask(15, p) == expected


def test_fraction_parser_is_not_eval():
    assert parse_fraction("1/4") == 0.25
    assert parse_fraction(0.5) == 0.5
    with pytest.raises(Exception):
        parse_fraction("__import__('os').system('true')")


def test_non_reentrant_wrapper_marks_a_single_block():
    import torch.nn as nn
    from fms_fsdp_b200.policies.ac_handler import is_checkpointed, non_reentrant_wrapper
    blk = nn.Linear(2, 2)
    assert not is_checkpointed(blk)
    assert non_reentrant_wrapper(blk) is blk and is_checkpointed(blk)


AC_FRACTIONS = ["1/7", "1/4", "1/3", "2/5", "1/2", "3/5", "2/3", "3/4", "9/10", "1"]
AC_DEPTHS = [10, 24, 32, 40, 48, 80]


def test_selection_equals_what_the_reference_install_wraps():
    """The unmodified reference ``apply_fsdp_checkpointing`` (torch ``checkpoint_wrapper``) was run on stacks of plain
    blocks for the depths of the model zoo and a sweep of fractions (oracle/make_golden.py); WHICH blocks it wrapped is
    recorded in tests/golden and must equal ``selection_mask``."""
    import gzip
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_selective_ac.json.gz")
    with gzip.open(path, "rt") as f:
        theirs = json.load(f)
    assert sorted(theirs) == sorted(f"{n}:{p}" for n in AC_DEPTHS for p in AC_FRACTIONS)
    for n in AC_DEPTHS:
        for p in AC_FRACTIONS:
            assert selection_mask(n, p) == theirs[f"{n}:{p}"], (n, p)
