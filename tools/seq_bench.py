"""Sequence mode throughput: S sequences advanced N scans in lockstep by lins_gpu_seq_step (host buffers in), against the
same feature logs through one C++ StateEstimator shim per sequence, plus the host StatePredictor::predict cost per scan.

    python tools/seq_bench.py --seqs 132,1000 --steps 20 --distinct 44

The logs are `--distinct` seeded simulated drives (config3), tiled to S sequences: a tiled sequence is computed again
from its own copy of the state, so the device does S sequences' work.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

capi, defs, synth = ge._pkg("capi"), ge._pkg("ctypes_defs"), ge._pkg("synth")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().split("\n")[0].split(", ") + ["?"])[:2] if q.returncode == 0 else ("unknown", "unknown")
    return name, power


def step_dict(logs, recs, t):
    scans = [synth.log_scan(l, r["handover_index"] + 1 + t) for l, r in zip(logs, recs)]
    step = dict(imu=np.concatenate([s["imu"] for s in scans]), imu_off=np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]))
    for c in defs.Batch.FIELDS:
        step[c] = np.concatenate([s[c] for s in scans])
        step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in scans])])
    return step


def run_device(logs, recs, steps):
    g = capi.LinsGpu()
    hs = [r["handover"] for r in recs]
    ho = {k: np.stack([h[k] for h in hs]) for k in ("filter_state", "filter_cov", "global_state", "imu_last")}
    for k in ("surf_map", "corner_map"):
        ho[k] = np.concatenate([h[k] for h in hs])
        ho[k + "_off"] = np.concatenate([[0], np.cumsum([len(h[k]) for h in hs])])
    g.seq_begin(defs.LinsSeqParams.shipped(), ho)
    wall, phases, iters, ran = 0.0, np.zeros(4), 0, 0
    for t in range(steps):
        sd = step_dict(logs, recs, t)
        t0 = time.perf_counter()
        g.seq_step(sd)  # (returns after its final stream synchronisation)
        wall += time.perf_counter() - t0
        phases += g.seq_phase_ms()
        d = g.seq_download()
        ok = d["status"] >= defs.SEQ_RAN
        ran += int(ok.sum())
        iters += int(d["results"]["iters"][ok].sum())
    g.close()
    return dict(seconds=wall, scans_per_s=ran / wall, eskf_iters_per_s=iters / wall, scans=ran,
                phase_ms_per_step=dict(zip(("predict", "ieskf", "fallback_check", "post_map"), (phases / steps).round(4).tolist())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", default="132,1000")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--distinct", type=int, default=44)
    a = ap.parse_args()
    name, power = gpu_info()
    logs = [synth.feature_log("config3", seed=5000 + i, n_scans=a.steps + 2) for i in range(a.distinct)]
    t0 = time.perf_counter()
    recs = [synth.replay_feature_log(l) for l in logs]
    shim_s = time.perf_counter() - t0
    shim_scans = sum(len(l["time"]) for l in logs)
    # steady state: the scans after the hand-over, each timed inside the replay (processImu calls + processFeatures)
    steady = [r["scan_s"][r["handover_index"] + 1:] for r in recs]
    steady_n, steady_s = sum(len(x) for x in steady), sum(float(x.sum()) for x in steady)
    L = synth.seq_lib()
    L.lins_bench_host_predict.restype = C.c_double
    L.lins_bench_host_predict.argtypes = [C.c_void_p, C.c_int, C.c_int]
    rows = np.ascontiguousarray(synth.log_scan(logs[0], 3)["imu"])
    per_call = L.lins_bench_host_predict(rows.ctypes.data, len(rows), 200)
    out = dict(metric="seq_mode", gpu=name, power_limit=power, steps=a.steps, distinct_logs=a.distinct,
               shim=dict(scans_per_s=shim_scans / shim_s, steady_scans_per_s=steady_n / steady_s,
                         note="one shim per sequence, run one after another; scans_per_s includes context creation and the first two "
                              "scans, steady_scans_per_s only the scans after the hand-over"),
               host_predict=dict(us_per_call=per_call * 1e6, calls_per_scan=len(rows), us_per_scan=per_call * len(rows) * 1e6))
    for S in [int(s) for s in a.seqs.split(",")]:
        idx = [i % a.distinct for i in range(S)]
        sl, sr = [logs[i] for i in idx], [recs[i] for i in idx]
        run_device(sl, sr, 2)  # warm-up: module load, allocations
        out[f"S{S}"] = run_device(sl, sr, a.steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
