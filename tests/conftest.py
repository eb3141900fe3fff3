import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90)")
    # the fp32 oracle is the numerical ground truth: no TF32 in its convolutions / matmuls when it runs on the GPU
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def parity_record(name: str, **values):
    """Append measured parity numbers to the JSON file named by SVR2_PARITY_RECORD (nothing is written when it is unset)."""
    import json
    path = os.environ.get("SVR2_PARITY_RECORD")
    if not path:
        return
    try:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        data = json.load(open(path)) if os.path.exists(path) else {}
        data[name] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in values.items()}
        json.dump(data, open(path, "w"), indent=1, sort_keys=True)
    except OSError:
        pass


@pytest.fixture(scope="session")
def pkg():
    from svr2_import import load_package
    return load_package()


@pytest.fixture(scope="session")
def svr2lib(pkg):
    import importlib
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")


@pytest.fixture(autouse=True)
def _release_engine_workspace():
    """The native runtimes keep one resident workspace per device (lib.workspace); tests that run the torch oracle on the
    same GPU right after need those bytes."""
    yield
    lib = sys.modules.get("comfyui_seedvr2_videoupscaler_b200.lib")
    if lib is not None:
        import torch
        if torch.cuda.is_available():
            lib.release_workspace()
