"""pytest configuration: registers the `gpu` marker and puts the repo root and
the product directory (`text-detection-ctpn_b200/`, whose name is not an
importable identifier) on sys.path."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "text-detection-ctpn_b200")
for p in (PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


def pytest_sessionstart(session):
    # the CPU oracle runs on torch-CPU: more than ~32 threads is much slower on many-core hosts
    try:
        import torch
        torch.set_num_threads(min(32, os.cpu_count() or 1))
    except Exception:
        pass
