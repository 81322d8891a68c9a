"""CPU: the ragged-batch ABI (ctpn_net_forward_ragged, ctpn_proposals_ragged) rejects bad arguments before any CUDA call,
the batch plan of Engine.detect_ragged (ragged_plan) is a partition with covering canvases, and tools/time_ragged.py's
dry run prints its record."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from ctpn_b200 import _native as N
from ctpn_b200.engine import ragged_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_symbols_are_in_the_abi():
    for name in ("ctpn_net_forward_ragged", "ctpn_proposals_ragged"):
        assert name in N.SIGNATURES and hasattr(N.lib, name)


@pytest.fixture
def net():
    h = C.c_void_p()
    N.check(N.lib.ctpn_net_create(C.byref(h), 2), "ctpn_net_create")
    yield h
    N.lib.ctpn_net_destroy(h)


def test_net_forward_ragged_rejects_bad_arguments(net):
    p = C.c_void_p(256)      # never dereferenced: validation comes first
    f = N.lib.ctpn_net_forward_ragged
    assert f(net, p, 0, None, 2, 64, 64, p, p, p, 1 << 20, None) == N.ERR_INVALID
    assert "null" in N.last_error()
    assert f(None, p, 0, p, 2, 64, 64, p, p, p, 1 << 20, None) == N.ERR_INVALID
    assert f(net, None, 0, p, 2, 64, 64, p, p, p, 1 << 20, None) == N.ERR_INVALID
    for B, H, W in ((0, 64, 64), (2, 15, 64), (2, 64, 8), (-1, 64, 64)):
        assert f(net, p, 0, p, B, H, W, p, p, p, 1 << 20, None) == N.ERR_INVALID
        assert "bad shape" in N.last_error()


def test_proposals_ragged_rejects_bad_arguments():
    p = C.c_void_p(256)
    f = N.lib.ctpn_proposals_ragged
    args = lambda feat, B, H, W: (p, 1, p, p, feat, B, H, W, 16, 12000, 1000, 0.7, 8.0, 0, p, p, p, p, 1 << 20, None)
    assert f(*args(None, 2, 4, 4)) == N.ERR_INVALID and "feat_hw" in N.last_error()
    for B, H, W in ((0, 4, 4), (2, 0, 4), (2, 4, -3)):
        assert f(*args(p, B, H, W)) == N.ERR_INVALID and "bad shape" in N.last_error()
    assert f(None, 1, p, p, p, 2, 4, 4, 16, 12000, 1000, 0.7, 8.0, 0, p, p, p, p, 1 << 20, None) == N.ERR_INVALID


def _random_shapes(seed, n):
    rs = np.random.RandomState(seed)
    shapes = [(int(rs.randint(16, 1200)), int(rs.randint(16, 1200))) for _ in range(n)]
    shapes += [(64, 64), (64, 64), (16, 16)]
    dtypes = [("|u1", "<f4")[int(rs.randint(2))] for _ in shapes]
    return shapes, dtypes


@pytest.mark.parametrize("seed,n,max_batch", [(0, 64, 32), (1, 100, 7), (2, 5, 1), (3, 40, 64)])
def test_ragged_plan_partitions_and_covers(seed, n, max_batch):
    shapes, dtypes = _random_shapes(seed, n)
    plan = ragged_plan(shapes, dtypes, max_batch)
    seen = [i for idx, _ in plan for i in idx]
    assert sorted(seen) == list(range(len(shapes)))                         # every index exactly once
    for idx, (H, W) in plan:
        assert 1 <= len(idx) <= max_batch
        assert len({dtypes[i] for i in idx}) == 1                           # no chunk mixes dtypes ...
        assert len({shapes[i][0] > shapes[i][1] for i in idx}) == 1         # ... or orientations
        assert all(shapes[i][0] <= H and shapes[i][1] <= W for i in idx)    # the canvas covers its members
        assert H == max(shapes[i][0] for i in idx) and W == max(shapes[i][1] for i in idx)
        assert [shapes[i] for i in idx] == sorted(shapes[i] for i in idx)   # sorted by (H, W) within the chunk
    # scattering the chunk results by index restores input order
    out = [None] * len(shapes)
    for idx, _ in plan:
        for i in idx:
            out[i] = shapes[i]
    assert out == shapes


def test_ragged_plan_is_deterministic_and_rejects_bad_batch():
    shapes, dtypes = _random_shapes(4, 30)
    assert ragged_plan(shapes, dtypes, 8) == ragged_plan(list(shapes), list(dtypes), 8)
    with pytest.raises(ValueError):
        ragged_plan(shapes, dtypes, 0)
    with pytest.raises(ValueError):
        ragged_plan(shapes, dtypes[:-1], 4)


def test_time_ragged_dry_run_prints_its_record():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "time_ragged.py"), "--dry-run"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    rec = json.loads(out.stdout.strip().splitlines()[-1])
    assert rec["dry_run"] and rec["images"] == 64 and sum(b[0] for b in rec["batches"]) == 64
    assert 0.0 <= rec["padded_fraction"] < 1.0 and 0 < rec["landscape"] < 64
    assert all(b[0] <= 32 and 16 <= b[1] <= 1000 and 16 <= b[2] <= 1000 for b in rec["batches"])
