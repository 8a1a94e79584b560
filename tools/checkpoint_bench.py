"""Saving and loading sequence-mode slots (lins_gpu_seq_save_size / _save / _load) at scale.

A bound run (lins_gpu_seq_open + lins_gpu_seq_map_open) of S slots tiles a few seeded VLP-16 raw-sweep drives
(synth.raw_log), each slot of a drive starting a few scans after the previous one, as tools/slam_bench.py does.  After
--steps steps of lins_gpu_seq_step_raw + lins_gpu_seq_map_step (the mapping windows near 50 key frames), it reports:
  - bytes per slot (mean and max), from the offsets lins_gpu_seq_save_size returns;
  - the wall time of saving every slot (lins_gpu_seq_save_size + lins_gpu_seq_save into a preallocated host buffer) and
    of loading them all into the fresh slots of a second bound run (lins_gpu_seq_load), each a host clock around calls
    that end in a stream synchronisation, median of --reps repetitions (every load goes to a newly opened run);
  - the median wall time of one step (seq_step_raw + seq_map_step) over --timed further steps, and the two ratios;
  - whether the loaded run's next step equals the source run's (downloads and mapper reports, byte for byte);
  - the card's name and power limit, read in the same run.

    python tools/checkpoint_bench.py [--slots 132,1000] [--drives 3] [--steps 170] [--timed 5] [--reps 5] [--phases 4]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="132,1000")
    ap.add_argument("--drives", type=int, default=3)
    ap.add_argument("--steps", type=int, default=170, help="steps before the save (window fill)")
    ap.add_argument("--timed", type=int, default=5, help="timed steps after the save")
    ap.add_argument("--reps", type=int, default=5, help="repetitions of the save and of the load")
    ap.add_argument("--phases", type=int, default=4, help="start offsets (scans) of the slots of one drive")
    a = ap.parse_args()
    from mapping_bench import _pkg, card

    capi, synth, defs = _pkg("capi"), _pkg("synth"), _pkg("ctypes_defs")
    synth.build()
    n_scans = a.steps + a.timed + 1 + a.phases
    logs = [synth.raw_log("config3", seed=21 + i, n_scans=n_scans) for i in range(a.drives)]
    model = defs.LinsLidarModel.vlp16()
    ip = defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))
    L = capi.lib()

    def clock(fn):
        t0 = time.perf_counter()
        out = fn()
        return out, 1e3 * (time.perf_counter() - t0)

    def bound_run(S):
        g = capi.LinsGpu()
        g.seq_open(defs.LinsSeqParams.shipped(), ip, S)
        g.seq_map_open()
        return g

    results = []
    for S in [int(x) for x in a.slots.split(",")]:
        drive = [s % a.drives for s in range(S)]
        phase = [(s // a.drives) % a.phases for s in range(S)]

        def step(g, k):
            lg = [logs[drive[s]] for s in range(S)]
            idx = [k + phase[s] for s in range(S)]
            imus = [l["imu"][l["imu_off"][i]:l["imu_off"][i + 1]] for l, i in zip(lg, idx)]
            st = dict(imu=np.concatenate(imus).reshape(-1, 7), imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32),
                      sweeps=[l["sweeps"][i] for l, i in zip(lg, idx)])
            si = np.array([l["imu_last"][i] for l, i in zip(lg, idx)])
            stamps = np.array([l["time"][i] for l, i in zip(lg, idx)])
            return lambda: (g.seq_step_raw(st, model=model, scan_imu=si), g.seq_map_step(stamps))[1]

        g = bound_run(S)
        fill = []
        for k in range(a.steps):
            reps, pub = step(g, k)()
            fill = [r.window_len for r in reps if r is not None and r.processed] or fill
            if k % 40 == 0:
                print(f"S = {S}: step {k} / {a.steps}", file=sys.stderr, flush=True)
        mask = np.ones(S, np.uint8)
        off = np.zeros(S + 1, np.uint64)
        g._ck(L.lins_gpu_seq_save_size(g.h, capi.ptr(mask), capi.ptr(off)))
        sizes = np.diff(off.astype(np.int64))
        buf = np.zeros(int(off[-1]), np.uint8)

        def save():
            g._ck(L.lins_gpu_seq_save_size(g.h, capi.ptr(mask), capi.ptr(off)))
            g._ck(L.lins_gpu_seq_save(g.h, capi.ptr(mask), capi.ptr(buf), capi.ptr(off)))

        t_save = [clock(save)[1] for _ in range(a.reps)]
        t_load, loaded = [], None
        for _ in range(a.reps):
            b = bound_run(S)
            t_load.append(clock(lambda: b._ck(L.lins_gpu_seq_load(b.h, capi.ptr(mask), capi.ptr(buf), capi.ptr(off))))[1])
            if loaded is not None:
                loaded.close()
            loaded = b
        # the loaded run's next step against the source's, then the timed steps of the source
        ra, _ = step(g, a.steps)()
        rb, _ = step(loaded, a.steps)()
        da, db = g.seq_download(), loaded.seq_download()
        equal = all(np.asarray(da[k]).tobytes() == np.asarray(db[k]).tobytes() for k in ("global_state", "filter_state", "filter_cov", "status"))
        equal &= all((x is None) == (y is None) and (x is None or bytes(x) == bytes(y)) for x, y in zip(ra, rb))
        t_step = [clock(step(g, a.steps + 1 + k))[1] for k in range(a.timed)]
        loaded.close()
        g.close()
        save_ms, load_ms, step_ms = float(np.median(t_save)), float(np.median(t_load)), float(np.median(t_step))
        res = dict(slots=S, window_fill_mean=round(float(np.mean(fill)), 1) if fill else 0.0, bytes_per_slot_mean=int(sizes.mean()),
                   bytes_per_slot_max=int(sizes.max()), total_mb=round(float(off[-1]) / 1e6, 1), save_ms=round(save_ms, 2),
                   load_ms=round(load_ms, 2), step_ms=round(step_ms, 2), save_over_step=round(save_ms / step_ms, 2),
                   load_over_step=round(load_ms / step_ms, 2), loaded_next_step_equal=bool(equal))
        results.append(res)
        print(json.dumps(res), file=sys.stderr)
    print(json.dumps(dict(card=card(), drives=a.drives, steps=a.steps, reps=a.reps, results=results)))
    return 0 if all(r["loaded_next_step_equal"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
