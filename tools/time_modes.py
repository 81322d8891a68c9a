"""Images/s of several arithmetic modes on the device-resident step that bench.py times (Engine.detect_packed on a resident
uint8 batch: conv stack, BiLSTM, heads, proposal layer), measured in one process with CUDA events.  The modes run in
alternating rounds after a warm-up of each, so that clock and neighbour drift hit all of them alike; the card's name and
power limit are read in the same run.

    python tools/time_modes.py --modes bf16x2,bf16x3,bf16x3p --batch 32 --rounds 5 --out profiles/time_modes_promoted.json
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "text-detection-ctpn_b200"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="bf16x2,bf16x3,bf16x3p")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--H", type=int, default=600)
    ap.add_argument("--W", type=int, default=900)
    ap.add_argument("--steps", type=int, default=5, help="timed steps per round")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per mode (at least 3)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps per mode before the first round")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="parse arguments and exit (no GPU)")
    a = ap.parse_args(argv)
    modes = a.modes.split(",")
    if a.rounds < 3:
        ap.error("--rounds: at least 3 rounds per mode")
    if a.dry_run:
        print(json.dumps({"modes": modes, "batch": a.batch, "H": a.H, "W": a.W, "steps": a.steps, "rounds": a.rounds,
                          "warmup": a.warmup, "out": a.out}))
        return None
    import numpy as np
    import torch
    from ctpn_b200 import Engine, synthetic as synth
    w = synth.make_weights(0)
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(100)
    images = torch.from_numpy(rs.randint(0, 256, size=(a.batch, a.H, a.W, 3), dtype=np.uint8)).to(dev)
    info = torch.tensor([[a.H, a.W, 1.0]] * a.batch, dtype=torch.float32, device=dev)
    engines = {m: Engine(w, mode=m) for m in modes}
    for m in modes:
        for _ in range(a.warmup):
            engines[m].detect_packed(images, info)
    torch.cuda.synchronize()
    ms = {m: [] for m in modes}
    for _ in range(a.rounds):
        for m in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                engines[m].detect_packed(images, info)
            e1.record()
            torch.cuda.synchronize()
            ms[m].append(e0.elapsed_time(e1) / a.steps)
    rec = {"card": card(), "batch": a.batch, "H": a.H, "W": a.W, "steps_per_round": a.steps, "rounds": a.rounds,
           "timed": "Engine.detect_packed on a device-resident uint8 batch, CUDA events, modes alternating per round",
           "modes": {}}
    for m in modes:
        med = float(np.median(ms[m]))
        rec["modes"][m] = {"ms_per_step": [round(t, 3) for t in ms[m]], "median_ms_per_step": round(med, 3),
                           "images_per_s": round(a.batch / (med / 1e3), 1)}
        print("%-8s median %.2f ms/step  %.1f images/s  (rounds %s)" % (m, med, a.batch / (med / 1e3),
                                                                       " ".join("%.2f" % t for t in ms[m])), flush=True)
    if "bf16x3" in modes and "bf16x3p" in modes:
        rec["bf16x3p_over_bf16x3"] = round(rec["modes"]["bf16x3p"]["images_per_s"] / rec["modes"]["bf16x3"]["images_per_s"], 3)
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)
    return rec


if __name__ == "__main__":
    main()
