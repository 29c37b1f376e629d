import os
import socket
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture
def narrow_model_factory():
    """1-wide Llama: module-structure tests are instant (reference tests/conftest.py:5-22)."""
    from fms_fsdp_b200.models.llama import LLaMA, LLaMAConfig

    def make(nlayers):
        return LLaMA(LLaMAConfig(src_vocab_size=1, emb_dim=1, nheads=1, nlayers=nlayers, multiple_of=1))
    return make


@pytest.fixture
def tiny_llama():
    from fms_fsdp_b200.models.llama import LLaMA
    from fms_fsdp_b200.utils.config_utils import get_model_config
    torch.manual_seed(0)
    m = LLaMA(get_model_config("llama2_tiny"))
    m.reset_parameters()
    return m
