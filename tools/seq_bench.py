"""Sequence mode throughput: S sequences advanced N scans in lockstep by lins_gpu_seq_step (host buffers in), against the
same feature logs through one C++ StateEstimator shim per sequence, plus the host StatePredictor::predict cost per scan.

    python tools/seq_bench.py --seqs 132,1000 --steps 20 --distinct 44
    python tools/seq_bench.py --queue --seqs 132,1000 --recordings 3 --reps 2

The logs are `--distinct` seeded simulated drives (config3), tiled to S sequences: a tiled sequence is computed again
from its own copy of the state, so the device does S sequences' work.  Prints one JSON line.

--queue: a replay job of R = --recordings x S recordings of spread lengths (seeded prefixes of the distinct logs) through
S slots, two ways, alternated --reps times in the same process:
  (a) open: lins_gpu_seq_open slots run every recording from its first scan, and a slot whose recording has ended is
      restarted (lins_gpu_seq_restart) with the next one on the following step;
  (b) begin: each recording's first two scans go through a host StateEstimator shim (the hand-over), then the recordings
      run in waves of S with lins_gpu_seq_begin, each wave as long as its longest recording.
Wall times cover the library calls only (building the step descriptors is not timed).  The shim hand-overs of (b) are
timed over the distinct logs (context creation + two scans each) and counted once per recording."""
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

capi, defs, synth, bag_replay = ge._pkg("capi"), ge._pkg("ctypes_defs"), ge._pkg("synth"), ge._pkg("bag_replay")


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


def cat_step(scans, present):
    step = dict(present=np.array(present, np.uint8), imu=np.concatenate([np.asarray(s["imu"]).reshape(-1, 7) for s in scans]),
                imu_off=np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]))
    for c in defs.Batch.FIELDS:
        step[c] = np.concatenate([s[c] for s in scans])
        step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in scans])])
    return step


def empty_scan(log):
    return dict(imu=np.zeros((0, 7)), imu_last=np.zeros(6), **{c: log[c][:0] for c in defs.Batch.FIELDS})


def queue_open(logs, jobs, S):
    """(a): every recording from its first scan in S opened slots, freed slots restarted with the next recording."""
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0)), S)
    wall, phases, steps, scans, n_first, n_second = 0.0, np.zeros(4), 0, 0, 0, 0
    for restart, who in bag_replay.slot_queue([n for _, n in jobs], S):
        sl, present, imu = [], [], np.zeros((S, 6))
        for j, w in enumerate(who):
            if w is None:
                sl.append(empty_scan(logs[0])); present.append(0)
                continue
            s = synth.log_scan(logs[jobs[w[0]][0]], w[1])
            sl.append(s); present.append(1); imu[j] = s["imu_last"]
        sd = cat_step(sl, present)
        t0 = time.perf_counter()
        if restart.any():
            g.seq_restart(restart)
        g.seq_step(sd, scan_imu=imu)
        wall += time.perf_counter() - t0
        phases += g.seq_phase_ms()
        st = g.seq_download()["status"]
        n_first += int((st == defs.SEQ_FIRST).sum()); n_second += int((st == defs.SEQ_SECOND).sum())
        steps += 1
        scans += sum(present)
    g.close()
    return dict(seconds=wall, scans=scans, steps=steps, scans_per_s=scans / wall, occupancy=scans / (steps * S),
                first_scans=n_first, second_scans=n_second, phase_ms_per_step=phase_dict(phases, steps),
                init_icp_share=float(phases[2] / phases.sum()))


def queue_begin(logs, recs, jobs, S):
    """(b): shim hand-overs (timed apart), then waves of S recordings from their third scan with lins_gpu_seq_begin."""
    g = capi.LinsGpu()
    wall, phases, steps, scans = 0.0, np.zeros(4), 0, 0
    for w0 in range(0, len(jobs), S):
        wave = jobs[w0:w0 + S]
        hs = [recs[li]["handover"] for li, _ in wave]
        ho = {k: np.stack([h[k] for h in hs]) for k in ("filter_state", "filter_cov", "global_state", "imu_last")}
        for k in ("surf_map", "corner_map"):
            ho[k] = np.concatenate([h[k] for h in hs])
            ho[k + "_off"] = np.concatenate([[0], np.cumsum([len(h[k]) for h in hs])])
        t0 = time.perf_counter()
        g.seq_begin(defs.LinsSeqParams.shipped(), ho)
        wall += time.perf_counter() - t0
        for t in range(max(n for _, n in wave) - 2):
            sl = [synth.log_scan(logs[li], 2 + t) if 2 + t < n else empty_scan(logs[li]) for li, n in wave]
            present = [int(2 + t < n) for _, n in wave]
            sd = cat_step(sl, present)
            t0 = time.perf_counter()
            g.seq_step(sd)
            wall += time.perf_counter() - t0
            phases += g.seq_phase_ms()
            steps += 1
            scans += sum(present)
    g.close()
    return dict(seconds=wall, scans=scans, steps=steps, scans_per_s=scans / wall, occupancy=scans / (steps * S),
                phase_ms_per_step=phase_dict(phases, steps))


def phase_dict(phases, steps):
    return dict(zip(("predict", "ieskf", "fallback_check_and_init_icp", "post_init_map"), (phases / max(steps, 1)).round(4).tolist()))


def main_queue(a, name, power):
    rng = np.random.default_rng(a.seed)
    logs = [synth.feature_log("config3", seed=7000 + i, n_scans=a.max_len) for i in range(a.distinct)]
    # the hand-over of (b): two scans through a fresh shim per distinct log, timed with its context creation
    recs, ho_s = [], []
    for l in logs:
        t0 = time.perf_counter()
        recs.append(synth.replay_feature_log(synth.make_log([synth.log_scan(l, k) for k in range(2)], l["lidar"])))
        ho_s.append(time.perf_counter() - t0)
    assert all(r["handover_index"] == 1 for r in recs)
    out = dict(metric="seq_queue", gpu=name, power_limit=power, distinct_logs=a.distinct, min_len=a.min_len, max_len=a.max_len,
               shim_handover_s=float(np.mean(ho_s)))
    for S in [int(s) for s in a.seqs.split(",")]:
        R = a.recordings * S
        jobs = [(int(rng.integers(a.distinct)), int(rng.integers(a.min_len, a.max_len + 1))) for _ in range(R)]
        res = dict(recordings=R, recording_scans=sum(n for _, n in jobs), open=[], begin=[])
        queue_open(logs, jobs[:S], S)  # warm-up: module load, allocations
        queue_begin(logs, recs, jobs[:S], S)
        for _ in range(a.reps):
            res["open"].append(queue_open(logs, jobs, S))
            b = queue_begin(logs, recs, jobs, S)
            b["handover_s"] = R * out["shim_handover_s"]
            b["scans_per_s_with_handover"] = res["recording_scans"] / (b["seconds"] + b["handover_s"])
            res["begin"].append(b)
        out[f"S{S}"] = res
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", default="132,1000")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--distinct", type=int, default=44)
    ap.add_argument("--queue", action="store_true", help="the replay-job comparison of open + restart against begin waves")
    ap.add_argument("--recordings", type=int, default=3, help="--queue: recordings per slot")
    ap.add_argument("--min-len", type=int, default=6)
    ap.add_argument("--max-len", type=int, default=30)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    name, power = gpu_info()
    if a.queue:
        return main_queue(a, name, power)
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
