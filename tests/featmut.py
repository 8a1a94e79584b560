"""Two mutated variants of tests/pyfront.py's feature selection — TEST INFRASTRUCTURE.

A hand-built scene proves that it reaches its condition when the reference's selection and a variant that gets the
condition wrong give different clouds:
  clip_to_ring:    suppression never leaves the ring's visited range (what a kernel that ran rings independently would do);
  suppress_fourth: the 4th flat point of a sextant is marked and suppressed like the first three.
The de-skew, curvature and occlusion stages are pyfront's (this repeats only its selection loop).
"""
import numpy as np

import pyfront


def select(seg, info, line_num, clip_to_ring=False, suppress_fourth=False, edge=0.5, surf=0.5):
    lm = pyfront.Lidar(line_num=line_num)
    und = pyfront.extract_features(seg, info, lm=lm)["undist"]
    n = len(seg)
    cap = max(lm.line_num * lm.scan_num, n + 16)
    r = np.zeros(cap, np.float32); r[:n] = info["range"]
    col = np.zeros(cap, np.int64); col[:n] = info["col"]
    ground = np.zeros(cap, np.uint8); ground[:n] = info["ground"]
    curv, picked, label = np.zeros(cap), np.zeros(cap, np.int64), np.zeros(cap, np.int64)
    sval, sind = np.zeros(cap), np.zeros(cap, np.int64)
    F = np.float32
    for i in range(5, n - 5):
        d = F(r[i - 5] + r[i - 4])
        for q in (-3, -2, -1):
            d = F(d + r[i + q])
        d = F(d - F(r[i] * F(10)))
        for q in (1, 2, 3, 4, 5):
            d = F(d + r[i + q])
        curv[i] = float(d) * float(d); sval[i] = curv[i]; sind[i] = i
    for i in range(5, n - 6):
        cd = abs(int(col[i + 1]) - int(col[i]))
        if cd < 10:
            if float(F(r[i] - r[i + 1])) > 0.3:
                picked[i - 5: i + 1] = 1
            elif float(F(r[i + 1] - r[i])) > 0.3:
                picked[i + 1: i + 7] = 1
        if float(abs(F(r[i - 1] - r[i]))) > 0.02 * float(r[i]) and float(abs(F(r[i + 1] - r[i]))) > 0.02 * float(r[i]):
            picked[i] = 1
    out = dict(sharp=[], less_sharp=[], flat=[], less_flat=[])

    def suppress(ind, lo, hi):
        picked[ind] = 1
        for l in range(1, 6):
            if ind + l >= cap or (clip_to_ring and ind + l > hi) or abs(int(col[ind + l]) - int(col[ind + l - 1])) > 10:
                break
            picked[ind + l] = 1
        for l in range(-1, -6, -1):
            if ind + l < 0 or (clip_to_ring and ind + l < lo) or abs(int(col[ind + l]) - int(col[ind + l + 1])) > 10:
                break
            picked[ind + l] = 1

    for i in range(line_num):
        s0, e0 = int(info["start_ring"][i]), int(info["end_ring"][i])
        ring_less = []
        for j in range(6):
            sp = (s0 * (6 - j) + e0 * j) // 6
            ep = (s0 * (5 - j) + e0 * (j + 1)) // 6 - 1
            if sp >= ep:
                continue
            o = np.argsort(sval[sp:ep], kind="stable")
            sval[sp:ep], sind[sp:ep] = sval[sp:ep][o], sind[sp:ep][o]
            big = 0
            for k in range(ep, sp - 1, -1):
                ind = int(sind[k])
                if picked[ind] == 0 and curv[ind] > edge and ground[ind] == 0:
                    big += 1
                    if big > 20:
                        break
                    label[ind] = 2 if big <= 2 else 1
                    if big <= 2:
                        out["sharp"].append(und[ind])
                    out["less_sharp"].append(und[ind])
                    suppress(ind, s0, e0 - 1)
            small = 0
            for k in range(sp, ep + 1):
                ind = int(sind[k])
                if picked[ind] == 0 and curv[ind] < surf and ground[ind] == 1:
                    label[ind] = -1
                    out["flat"].append(und[ind])
                    small += 1
                    if small >= 4:
                        if suppress_fourth:
                            suppress(ind, s0, e0 - 1)
                        break
                    suppress(ind, s0, e0 - 1)
            for k in range(sp, ep + 1):
                if label[k] <= 0:
                    ring_less.append(und[k])
        out["less_flat"].extend(list(pyfront.voxel_grid(np.asarray(ring_less, np.float32).reshape(-1, 4))))
    return {k: np.asarray(v, np.float32).reshape(-1, 4) for k, v in out.items()}


def differs(a, b):
    return any(a[k].shape != b[k].shape or not np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)) for k in a)
