import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")
    # the PyTorch fp32 references of the kernel tests must be fp32: by default cuDNN runs fp32 convolutions in TF32 on a GPU
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def golden_index():
    with open(os.path.join(GOLDEN, "index.json")) as f:
        return json.load(f)


def golden_schema(variant):
    with open(os.path.join(GOLDEN, f"{variant}.schema.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
