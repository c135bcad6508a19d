"""Per-panel timeline of the reduced-system Cholesky (csrc/chol.cu) inside one C3 LM solve, from a torch.profiler trace.

   python tools/chol_timeline.py [--iters 10] [--trace FILE.json]

Profiles one `lm_solve` of bench.py's C3 problem (after one warm-up solve) and prints, per panel step b (median over
the factorisations of the solve, plus the last factorisation in full):
  grid      CTAs of chol_panel_kernel b
  panel     start to end of the panel kernel (us); a kernel starts with its first CTA, so panel CTAs that wait for an
            SM held by update CTAs lengthen this column, not the gap
  gap       end of panel b to start of panel b+1 (us)
  upd@start chol_update_kernel launches still running when panel b starts, and how long the last of them still runs
The factorisation span is the first panel's start to the end of the last chol_* kernel before the next factorisation.
Times are device timestamps of the trace; the profiler adds a little overhead per launch, so take end-to-end numbers
from bench.py and tools/microbench.py chol."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def kernels_from_trace(path):
    ev = json.load(open(path))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    out = []
    for e in ev:
        if e.get("cat") == "kernel" and e.get("ph") == "X":
            grid = e.get("args", {}).get("grid", [0, 0, 0])
            out.append({"name": e["name"], "ts": float(e["ts"]), "end": float(e["ts"]) + float(e["dur"]),
                        "grid": int(grid[0]) if grid else 0})
    out.sort(key=lambda k: k["ts"])
    return out


def timeline(kernels, nblk):
    panels = [k for k in kernels if "chol_panel_kernel" in k["name"]]
    updates = [k for k in kernels if "chol_update_kernel" in k["name"]]
    if not panels or len(panels) % nblk:
        raise RuntimeError(f"{len(panels)} panel kernels in the trace, not a multiple of {nblk} panels per factorisation")
    facts = []
    for f in range(len(panels) // nblk):
        ps = panels[f * nblk:(f + 1) * nblk]
        lim = panels[(f + 1) * nblk]["ts"] if (f + 1) * nblk < len(panels) else float("inf")
        ups = [u for u in updates if ps[0]["ts"] <= u["ts"] < lim]
        end = max([p["end"] for p in ps] + [u["end"] for u in ups])
        steps = []
        for b, p in enumerate(ps):
            running = [u for u in ups if u["ts"] < p["ts"] < u["end"]]
            steps.append({"grid": p["grid"], "panel": p["end"] - p["ts"],
                          "gap": (ps[b + 1]["ts"] - p["end"]) if b + 1 < nblk else end - p["end"],
                          "upd_running": len(running), "upd_ctas": sum(u["grid"] for u in running),
                          "upd_tail": max([u["end"] - p["ts"] for u in running], default=0.0)})
        facts.append({"span": end - ps[0]["ts"], "steps": steps,
                      "panel_sum": sum(s["panel"] for s in steps), "update_kernels": len(ups),
                      "update_busy": sum(u["end"] - u["ts"] for u in ups)})
    return facts


def report(facts, nblk):
    def med(key, b):
        return float(np.median([f["steps"][b][key] for f in facts]))
    print(f"{len(facts)} factorisations of {nblk} panels; span median {np.median([f['span'] for f in facts]):.1f} us "
          f"(min {min(f['span'] for f in facts):.1f}), panel kernels median sum {np.median([f['panel_sum'] for f in facts]):.1f} us, "
          f"update kernels {facts[-1]['update_kernels']} per factorisation")
    print("  step  grid  panel_us  gap_us  upd@start  upd_ctas  upd_tail_us   (median over factorisations)")
    for b in range(nblk):
        print(f"  {b:4d}  {int(med('grid', b)):4d}  {med('panel', b):8.1f}  {med('gap', b):6.1f}  {med('upd_running', b):9.0f}"
              f"  {med('upd_ctas', b):8.0f}  {med('upd_tail', b):11.1f}")
    last = facts[-1]
    print(f"  last factorisation: span {last['span']:.1f} us; per step panel/gap us: " +
          " ".join(f"{s['panel']:.1f}/{s['gap']:.1f}" for s in last["steps"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--trace", default=None, help="keep the chrome trace here (default: a temporary file)")
    args = ap.parse_args()
    from bench import make_problem, S_FRAMES
    from vggsfm_b200 import bundle_adjustment as ba
    dev = torch.device("cuda:0")
    sc, extr, K, extra, pts = make_problem()
    model, mode = ba.SIMPLE_RADIAL, ba.INTR_SHARED
    intr = np.zeros((S_FRAMES, 4))
    intr[:, 0], intr[:, 1], intr[:, 2], intr[:, 3] = K[0, 0, 0], K[0, 0, 2], K[0, 1, 2], extra[0, 0]
    t = lambda a, dt=None: (torch.from_numpy(np.ascontiguousarray(a)).to(dt) if dt else torch.from_numpy(np.ascontiguousarray(a))).to(dev).contiguous()
    uv, mask = t(sc.tracks, torch.float32), t(sc.mask.astype(np.uint8))
    poses, intr_t, X = t(extr), t(intr), t(pts)
    opt = ba.default_options()
    opt.max_num_iterations = args.iters
    opt.gradient_tolerance = 0.0
    run = lambda: ba.lm_solve(uv, mask, poses.clone(), intr_t.clone(), X.clone(), model, mode, options=opt)
    run()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        s = run()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = args.trace or os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        kernels = kernels_from_trace(path)
    dc, ns = ba.dims(model, mode)
    n = S_FRAMES * dc + ns + 1                       # the bordered reduced system
    nblk = (n + 127) // 128
    tot = {}
    for k in kernels:
        tot[k["name"].split("(")[0].split("<")[0]] = tot.get(k["name"].split("(")[0].split("<")[0], 0.0) + k["end"] - k["ts"]
    busy = sum(tot.values())
    print(f"C3 lm_solve, {s.iterations} LM iterations, order {n}: device kernel time {busy / 1e3:.2f} ms; " +
          ", ".join(f"{k.split('::')[-1]} {v / busy * 100:.0f}%" for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:6]))
    report(timeline(kernels, nblk), nblk)


if __name__ == "__main__":
    main()
