"""Sequence mode feeding its mapping nodes (lins_gpu_seq_map_step) against today's composition on the host.

S slots tile a few seeded VLP-16 raw-sweep drives (synth.raw_log), each slot starting its drive a few scans after the
previous slot of the same drive (as tools/mappers_bench.py tiles its drives).  Two arms run the same sweeps, alternated
step by step in one process:
  (a) bound:   lins_gpu_seq_step_raw, then lins_gpu_seq_map_step (publish + mapping on the device clouds);
  (b) host:    an unbound context running the same lins_gpu_seq_step_raw, then seq_download + seq_download_init +
               seq_download_maps + project_scans of the NaN-filtered sweeps for the outlier clouds, publishTopics' rule
               in numpy (tests/slamref.py) and lins_gpu_mappers_step from host buffers.
The host arm runs the first --check slots (all of them when S <= --check), with the same drives and phases: slots are
independent, so each of its slots must equal the bound run's slot of the same index.  Its times are per step of those
slots only.
Per arm: ms per step of the sequence step and of the publish + mapping part (host clock around calls that end in a
stream synchronisation), mapping cycles/s (processed cycles over the publish + mapping time), and the payload bytes each
arm moves per step (H2D / D2H of clouds, states and counts, computed from array sizes).  The first --skip steps are not
timed (initialisation and the mapping windows filling); the window fill of the timed steps is reported.  Every step the
two arms' published flags and reports must be byte-equal, and at the end every slot's mapper download; the result says
whether they were.  The card's name and power limit are read in the same run.

    python tools/slam_bench.py [--slots 132,1000] [--drives 3] [--scans 180] [--skip 160] [--phases 4] [--check 132]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="132,1000")
    ap.add_argument("--drives", type=int, default=3)
    ap.add_argument("--scans", type=int, default=180, help="scans per drive")
    ap.add_argument("--skip", type=int, default=160, help="untimed steps (initialisation, window fill)")
    ap.add_argument("--check", type=int, default=132, help="slots the host arm runs and checks")
    ap.add_argument("--phases", type=int, default=4, help="start offsets (scans) of the slots of one drive")
    a = ap.parse_args()
    import slamref as sr
    from mapping_bench import _pkg, card

    capi, synth, defs = _pkg("capi"), _pkg("synth"), _pkg("ctypes_defs")
    synth.build()
    logs = [synth.raw_log("config3", seed=21 + i, n_scans=a.scans) for i in range(a.drives)]
    finite = [[s[np.isfinite(s[:, :3]).all(1)] for s in l["sweeps"]] for l in logs]
    n_steps = a.scans - a.phases
    model = defs.LinsLidarModel.vlp16()
    ip = defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))

    def pts(xyzi):
        x = np.asarray(xyzi, np.float32).reshape(-1, 4)
        return defs.make_points(x[:, :3], x[:, 3])

    def xyzi(p):
        return np.stack([p["x"], p["y"], p["z"], p["intensity"]], 1).astype(np.float32) if len(p) else np.zeros((0, 4), np.float32)

    def clock(fn):
        t0 = time.perf_counter()
        out = fn()
        return out, 1e3 * (time.perf_counter() - t0)

    results, all_equal = [], True
    for S in [int(x) for x in a.slots.split(",")]:
        drive = [s % a.drives for s in range(S)]
        phase = [(s // a.drives) % a.phases for s in range(S)]
        C = min(S, a.check)
        ga, gb = capi.LinsGpu(), capi.LinsGpu()
        ga.seq_open(defs.LinsSeqParams.shipped(), ip, S)
        gb.seq_open(defs.LinsSeqParams.shipped(), ip, C)
        ga.seq_map_open()
        gb.mappers_open(C)
        pub = sr.Publisher(C)
        t_seq = {"a": [], "b": []}
        t_map = {"a": [], "b": []}
        cycles, cycles_b, fill, bytes_a, bytes_b = [], [], [], [], []
        last = [None] * S
        equal = True
        for k in range(n_steps):
            sweeps = [logs[drive[s]]["sweeps"][k + phase[s]] for s in range(S)]
            imus = [logs[drive[s]]["imu"][logs[drive[s]]["imu_off"][k + phase[s]]:logs[drive[s]]["imu_off"][k + phase[s] + 1]] for s in range(S)]
            step = dict(imu=np.concatenate(imus).reshape(-1, 7), imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32),
                        sweeps=sweeps)
            si = np.array([logs[drive[s]]["imu_last"][k + phase[s]] for s in range(S)])
            stamps = np.array([logs[drive[s]]["time"][k + phase[s]] for s in range(S)])
            sweep_bytes = 32 * sum(len(w) for w in sweeps) + step["imu"].nbytes + si.nbytes
            # (a) bound
            _, ms = clock(lambda: ga.seq_step_raw(step, model=model, scan_imu=si))
            t_seq["a"].append(ms)
            (reps_a, pub_a), ms = clock(lambda: ga.seq_map_step(stamps))
            t_map["a"].append(ms)
            # (b) today's composition, on the first C slots
            before = gb.seq_download_init()["fusion_status"]
            io = step["imu_off"]
            step_b = dict(imu=step["imu"][: io[C]], imu_off=io[: C + 1], sweeps=sweeps[:C])
            _, ms = clock(lambda: gb.seq_step_raw(step_b, model=model, scan_imu=si[:C]))
            t_seq["b"].append(ms)

            def host_part():
                d, _ = gb.seq_download(), gb.seq_download_init()
                maps = gb.seq_download_maps()
                proj = gb.project_scans([finite[drive[s]][k + phase[s]] for s in range(C)], model=model)
                steps, moved = [None] * C, [0, 0]
                moved[1] += sum(32 * len(maps[c][s]) for c in ("surf_map", "corner_map", "surf_tree", "corner_tree") for s in range(C))
                moved[1] += C * (19 * 8 * 2 + 324 * 8 + 64) + sum(16 * len(p["outlier"]) + 16 * len(p["seg"]) for p in proj)
                moved[0] += 32 * sum(len(f) for f in proj)
                for s in range(C):
                    out = pub.step(s, before[s], int(d["status"][s]), d["global_state"][s], xyzi(maps["corner_map"][s]), xyzi(maps["surf_map"][s]),
                                   proj[s]["outlier"])
                    if out is not None:
                        steps[s] = (stamps[s], out[0][3:], out[0][:3], pts(out[1]), pts(out[2]), pts(out[3]))
                        moved[0] += 32 * (len(out[1]) + len(out[2]) + len(out[3])) + 8 * 8
                return gb.mappers_step(steps), steps, moved

            (reps_b, steps_b, moved), ms = clock(host_part)
            t_map["b"].append(ms)
            ok = pub_a[:C].tolist() == [int(x is not None) for x in steps_b]
            ok &= all(bytes(reps_a[s]) == bytes(reps_b[s]) for s in range(C) if pub_a[s])
            equal &= ok
            for s in range(S):
                if pub_a[s] and reps_a[s].processed:  # (a download is sized by the last processed cycle's report)
                    last[s] = reps_a[s]
            n_proc = sum(1 for s in range(S) if pub_a[s] and reps_a[s].processed)
            cycles.append(n_proc)
            cycles_b.append(sum(1 for s in range(C) if pub_a[s] and reps_a[s].processed))
            fill.append(float(np.mean([r.window_len for r in reps_a if r is not None and r.processed] or [0])))
            # payload bytes per step: sweeps + IMU up and the step's own read-backs in both arms; (a) adds the global
            # states and outlier counts it reads back; (b) adds what host_part moves
            bytes_a.append((sweep_bytes, S * (20 * 8 + 8)))
            bytes_b.append((sweep_bytes * C / S + moved[0], moved[1]))
            if k % 20 == 0:
                print(f"S = {S}: step {k} / {n_steps}, window fill {fill[-1]:.1f}, equal so far {equal}", file=sys.stderr, flush=True)
        for s in range(C):
            if last[s] is not None:
                equal &= ga.mappers_download(s, last[s])[0].tobytes() == gb.mappers_download(s, last[s])[0].tobytes()
        all_equal &= equal
        tm = slice(a.skip, None)
        res = dict(slots=S, timed_steps=n_steps - a.skip, window_fill_mean=round(float(np.mean(fill[tm])), 1),
                   processed_per_step=round(float(np.mean(cycles[tm])), 1), bit_equal=bool(equal), host_arm_slots=C)
        for arm, b, cyc in (("bound", bytes_a, cycles), ("host", bytes_b, cycles_b)):
            key = "a" if arm == "bound" else "b"
            seq_ms, map_ms = float(np.median(t_seq[key][tm])), float(np.median(t_map[key][tm]))
            res[arm] = dict(seq_step_ms=round(seq_ms, 2), publish_map_ms=round(map_ms, 2),
                            cycles_per_s=round(float(np.mean(cyc[tm])) / map_ms * 1e3, 1) if map_ms else 0.0,
                            h2d_mb=round(float(np.mean([x[0] for x in b[a.skip:]])) / 1e6, 2),
                            d2h_mb=round(float(np.mean([x[1] for x in b[a.skip:]])) / 1e6, 2))
        results.append(res)
        print(json.dumps(res), file=sys.stderr)
        ga.close(); gb.close()
    print(json.dumps(dict(card=card(), drives=a.drives, scans=a.scans, skip=a.skip, all_bit_equal=bool(all_equal), results=results)))
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
