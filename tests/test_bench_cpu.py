"""CPU: the arithmetic bench.py reports against -- algorithmic FLOPs per image (SURVEY.md App. A.1), the source hash that gates
a committed ncu traffic figure -- and its configurations following BASELINE.json."""
import glob
import json
import os

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_algorithmic_work_matches_the_survey_tables():
    a = bench.work_per_image(600, 900)                       # cfgA: 37 x 56 feature map
    assert (a["fh"], a["fw"], a["cells"]) == (37, 56, 2072)
    assert abs(a["conv1_1"] / 1e9 - 1.866) < 1e-3
    assert abs((a["conv1_1"] + a["conv3x3"]) / 1e9 - 339.130) < 5e-3
    assert abs(a["xproj"] / 1e9 - 2.173) < 1e-3 and abs(a["recurrent"] / 1e9 - 0.543) < 1e-3 and abs(a["fc"] / 1e9 - 0.543) < 1e-3
    b = bench.work_per_image(1200, 1600)                     # cfgB: 75 x 100
    assert (b["fh"], b["fw"]) == (75, 100)
    assert abs((b["conv1_1"] + b["conv3x3"]) / 1e9 - 1209.876) < 2e-2
    c = bench.work_per_image(900, 600)                       # the transposed shape of config 5
    assert (c["fh"], c["fw"]) == (56, 37)


def test_configs_follow_baseline_json():
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    assert len(base["configs"]) == 5
    assert bench.CONFIGS[2]["batch"] == 32 and bench.CONFIGS[2]["shapes"] == [(600, 900)] and bench.CONFIGS[2]["detect"] == "H"
    assert bench.CONFIGS[3]["mode"] == "bf16" and "bf16" in base["configs"][2]
    assert bench.CONFIGS[4]["batch"] == 32 and bench.CONFIGS[4]["shapes"] == [(1200, 1600)] and "1200" in base["configs"][3]
    assert bench.CONFIGS[5]["detect"] == "O" and len(bench.CONFIGS[5]["shapes"]) == 2 and "oriented" in base["configs"][4]
    assert bench.MODES[bench.FP32_MODE]["units"] in (2.0, 3.0)          # a float32-faithful mode, never plain bf16


def test_traffic_files_are_stamped_with_a_source_hash():
    sha = bench.sources_sha256()
    assert len(sha) == 64 and sha == bench.sources_sha256()
    # every committed capture (tools/ncu_traffic.py) carries the hash of the sources it was taken from
    for f in glob.glob(os.path.join(ROOT, "profiles", "conv_traffic_cfg*_*.json")):
        t = json.load(open(f))
        assert t["launches"] == 13 and len(t["sources_sha256"]) == 64 and t["dram_bytes_per_step"] > 1e10
        # 20.6 GB algorithmic per 32-image step at 4 B per activation element: the capture must be within 5 % of it
        assert abs(t["dram_bytes_per_step"] / 20.6e9 - 1.0) < 0.05
