"""Per-phase cycle breakdown of the fused kernel (diagnostics; run on a GPU box).
CTA-cycles: every CTA's thread 0 clocks the phases of its lockstep pass over the resident units (slots)."""
import importlib, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
config = sys.argv[2] if len(sys.argv) > 2 else "config3"
b = synth.generate(config, n=n, seed0=1000)
g = capi.LinsGpu(defs.LinsParams.shipped())
g.batch_upload(b); g.batch_run(); g.sync()
g.phase_cycles(enable=True)
g.batch_run(); g.sync()
t = g.phase_cycles(enable=False, read=True)
_, _, res, _ = g.batch_download(states=False, covs=False)
its = int(res["iters"].sum())
names = {1: "claim units (loop top)", 0: "prologues (prior, index build, staging)", 3: "de-skew + certificates (P1)", 4: "closest-point searches (P2)",
         5: "walk windows + walks (P3+P4)", 6: "residual + fold", 18: "tail: sums + A6 (slot 0's warp)", 19: "tail: M6 + LU", 21: "tail: K x, norms",
         23: "tail: logic + boxPlus", 25: "tail: next consts + boxMinus", 8: "wait for the other tails", 9: "exit cov + outputs"}
for k in (3, 4, 5, 6):  # passes with / without a unit in its first pass are clocked separately (+32)
    t[k] += t[k + 32]
tot = sum(t[k] for k in names)
print(f"units {n} iterations {its}  total CTA-cycles {tot:.3e}  per unit-iteration {tot/its:.0f} cycles")
for k, nm in names.items():
    print(f"  {nm:42s} {100*t[k]/tot:5.1f}%   {t[k]/its:9.0f} cycles per unit-iteration")
import torch
n_cta = torch.cuda.get_device_properties(0).multi_processor_count  # one CTA per SM
print("CTA busy: mean %.3e max %.3e (end-of-grid tail %.1f%%)" % (t[26]/n_cta, t[27], 100*(1-t[26]/n_cta/max(t[27],1))))
print("work lists per unit-iteration: closest-point searches %.1f (ring-bins per search %.1f), walk searches %.1f (ring-bins per search %.1f)" % (
    t[10]/its, t[12]/max(t[10],1), t[11]/its, t[13]/max(t[11],1)))
print("passes with a first-pass unit: %d (%.2f units resident), cycles per pass: P1 %.0f  P2 %.0f  P3+P4 %.0f  residual %.0f" % (
    t[62], t[63]/max(t[62],1), t[35]/max(t[62],1), t[36]/max(t[62],1), t[37]/max(t[62],1), t[38]/max(t[62],1)))
print("other passes:                   %d (%.2f units resident), cycles per pass: P1 %.0f  P2 %.0f  P3+P4 %.0f  residual %.0f" % (
    t[30], t[31]/max(t[30],1), (t[3]-t[35])/max(t[30],1), (t[4]-t[36])/max(t[30],1), (t[5]-t[37])/max(t[30],1), (t[6]-t[38])/max(t[30],1)))
# certificates of seeded queries (lins_assoc.cuh, kCertSlots = 40): two 32-bit counts per slot, closest point low, walks high
cert = [[(int(t[40 + k]) >> (32 * h)) & 0xffffffff for k in range(8)] for h in (0, 1)]
for h, nm in ((0, "closest point"), (1, "walks")):
    c = cert[h]
    print(f"certificates, {nm:13s}: checked {c[0]}  accepted {c[1]} ({100*c[1]/max(c[0],1):.1f}%, by a swap {c[7]})  failed: runner-up wins {c[2]}"
          f"  bound {c[3]}  left the gate {c[4]}  slack used up {c[5]};  failed but a stored front-runner was the answer {c[6]}")
print(f"  checked = accepted + failed: {all(c[0] == c[1] + sum(c[2:6]) for c in cert)}")
# later passes by their number of searches (kPassSlots = 48)
later = max(int(t[30]), 1)
for nm, base, labels, ph in (("closest-point", 48, ("0", "1-16", ">16"), "P2"), ("walk", 54, ("0", "1-16", "17-32", ">32"), "P3+P4")):
    nb = len(labels)
    print(f"later passes by {nm} searches: " + "  ".join(
        f"{lab}: {100*t[base+b]/later:.1f}% ({t[base+nb+b]/max(t[base+b],1):.0f} {ph} cycles)" for b, lab in enumerate(labels)))
