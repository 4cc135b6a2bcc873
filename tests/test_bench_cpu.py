"""bench.py's CPU arm (`--impl reference`) end to end on a small clip: the reference encoders start, the observing shim publishes progress, one JSON line with the contract's
keys comes out.  (The GPU arm needs a GPU; its workload capture and job parsing are covered by tests/test_rdo_jobs.py.)"""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs = pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "Thorenc_capture")), reason="oracle/_ref not built")


@needs
def test_reference_arm_prints_a_contract_line(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1", "--cpu-procs", "2", "--size", "640x384",
                        "--cpu-slice", "1.5", "--cache", str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1500:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    assert d["impl"] == "reference" and d["unit"] == "Mpixel/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": "Mpixel/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    c = d["cpu_baseline"]
    assert c["kind"] == "reference" and c["cores"] == 2 and c["value"] == d["value"] and "sample" in c
    assert d["steps"] == 2 and len(c["slices_rd_loop_mpixel_s"]) == 2          # steady-state slices, not the whole-run fallback
    assert 1.0 < c["effective_cores"] <= 2.05
    # the GPU arm would reuse this measurement of the box
    assert os.path.exists(os.path.join(str(tmp_path), "cpu_arm_hdb_640x384_17", "last_result.json"))
