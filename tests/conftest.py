import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


# the tests drive devices themselves (several GPUs in one process where the box has them): the library must not narrow
# CUDA_VISIBLE_DEVICES to its one-shot-CLI default before CUDA initialises
os.environ.setdefault("KREP_B200_KEEP_VISIBLE", "1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
