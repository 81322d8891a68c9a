#!/usr/bin/env python
"""Proposal-layer checks under the test library's NMS switches, run as subprocesses by tests/test_proposal_paths_gpu.py:
CTPN_COLUMN_GATHER and CTPN_GENERIC_NMS are read once per process.  Each sub-command prints one JSON line
{"ok": bool, ...} as its last line of stdout.

    mixed         the 62 x 37 three-image batch of proposal_cases.mixed_batch at NMS thresholds 0.7 and 0.03
    column_pairs  the borderline column pairs of proposal_cases.column_pairs at thresholds 0.7 and 0.5

    CTPN_B200_LIB=dbg CTPN_COLUMN_GATHER=1 python tests/proposal_checks.py mixed
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import proposal_cases as P  # noqa: E402


def _run(eng, cls, bbox, info, cfg):
    from test_proposal_paths_gpu import run_layer
    rois, index, count, column = run_layer(eng, cls, bbox, info, cfg)
    bad = []
    for b in range(cls.shape[0]):
        want, idx = P.oracle_layer(cls[b:b + 1], bbox[b:b + 1], info[b:b + 1], cfg)
        bad += ["image %d: %s" % (b, m) for m in P.layer_mismatches(rois[b], index[b], count[b], want, idx)]
    return bad, column


def main():
    from ctpn_b200 import _native as N
    from ctpn_b200.engine import Engine
    cmd = sys.argv[1]
    assert N.DEBUG_LIB, "run with CTPN_B200_LIB=dbg: the NMS switches exist in the test library only"
    env = {k: os.environ[k] for k in ("CTPN_COLUMN_GATHER", "CTPN_GENERIC_NMS") if k in os.environ}
    eng = Engine(None)
    res = dict(cmd=cmd, env=sorted(env), runs=[])
    ok = True
    if cmd == "mixed":
        runs = [(t, P.mixed_batch()) for t in (0.7, 0.03)]
    elif cmd == "column_pairs":
        runs = [(t, P.column_pair_heads(P.column_pairs(t))[:3]) for t in (0.7, 0.5)]
    else:
        raise SystemExit("unknown command %r" % cmd)
    for thresh, (cls, bbox, info) in runs:
        path = P.dispatch(cls.shape[1], cls.shape[2], lib=env)
        bad, column = _run(eng, cls, bbox, info, dict(RPN_NMS_THRESH=thresh))
        res["runs"].append(dict(thresh=thresh, path=path, column_kernel=column, mismatches=bad[:8]))
        ok = ok and not bad and column == (path[0] != "generic-all")
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
