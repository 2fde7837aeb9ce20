import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with -m gpu)")
    if os.environ.get("THB_SIMT_EMULATION") == "1":
        # opt-in DRY RUN of the GPU tests on the host emulation of the kernels (tests/simt/emulation_mode.py); never set by the driver
        import importlib.util
        spec = importlib.util.spec_from_file_location("emulation_mode", os.path.join(ROOT, "tests", "simt", "emulation_mode.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.enable()
