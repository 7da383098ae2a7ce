import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


# Worst observed parity errors of the -m gpu run: tests call ``record_error``; with NNAB_ERROR_LOG_DIR set
# the session writes them to $NNAB_ERROR_LOG_DIR/parity_errors.json.
PARITY_ERRORS = {}


def record_error(test, case, **fields):
    PARITY_ERRORS.setdefault(test, {})[case] = fields


def pytest_sessionfinish(session, exitstatus):
    out = os.environ.get("NNAB_ERROR_LOG_DIR")
    if not PARITY_ERRORS or not out:
        return
    import json

    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, "parity_errors.json")
    merged = {}
    if os.path.exists(path):
        try:
            with open(path) as f:
                merged = json.load(f)
        except Exception:  # noqa: BLE001
            merged = {}
    for k, v in PARITY_ERRORS.items():
        merged.setdefault(k, {}).update(v)
    with open(path, "w") as f:
        json.dump(merged, f, indent=1, sort_keys=True)
