#!/usr/bin/env python
"""Time the two-view stage (csrc/twoview.cu, vgg_estimate_fundamental) at the production shape: 400 pairs x 4096
matches, T = 4096 minimal samples, lo = 300, fmat_thres 4 (threshold 16 px^2), 30 % invisible, 5 % outliers.

Prints one JSON line: ms per call (CUDA events over `--iters` calls after `--warmup`), Sampson evaluations per second,
the FP64 bound of the minimal + scoring phase at the SM clock sampled during the timed calls (NVML), and the split of
kernel time between the phases (torch.profiler, in a separate pass after the timed one).

    python tools/twoview_bench.py [--pairs 400 --points 4096 --trials 4096 --lo 300 --iters 5 --warmup 2]

``--estimator poselib`` times the default configuration's stage instead (csrc/twoview_msac.cu,
vgg_estimate_fundamental_msac: LO-MSAC with PoseLib's stopping rule, max_iterations 20000, min_iterations 1000) on the
same workload, and adds the histogram of RANSAC iterations per pair, the LO runs per pair, the card name and power
limit (NVML, read in the same call), and the CPU oracle's time on a few pairs (``--oracle-pairs``; the restatement,
not PoseLib).
"""
import argparse
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# FP64 instructions (DFMA / DMUL) one Sampson evaluation issues in tv_minimal_kernel: 16 in sampson_parts + the
# prefilter's product; the division only runs near the threshold
FP64_OPS_PER_EVAL = 17
FP64_OPS_PER_CLK_PER_SM = 64       # H100 SXM: 64 FP64 FMA per clock per SM outside the tensor cores
PHASES = {"tv_minimal_kernel": "minimal+scoring", "tv_topk_kernel": "lo", "tv_lo_kernel": "lo",
          "tv_select_kernel": "select"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=400)
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--trials", type=int, default=4096)
    ap.add_argument("--lo", type=int, default=300)
    ap.add_argument("--max-error", type=float, default=4.0)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--estimator", choices=["7pt8pt", "poselib"], default="7pt8pt")
    ap.add_argument("--max-iterations", type=int, default=20000)
    ap.add_argument("--oracle-pairs", type=int, default=2)
    a = ap.parse_args()
    if a.estimator == "poselib":
        return bench_poselib(a)
    import torch
    from bench import ClockSampler
    from vggsfm_b200 import two_view as tv
    from vggsfm_b200.synthetic import make_scene
    if not torch.cuda.is_available():
        raise SystemExit("twoview_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    B, N = a.pairs, a.points
    sc = make_scene(B + 1, N, seed=0, invisible_frac=0.3, outlier_frac=0.05)
    p1 = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(sc.tracks[:1], (B, N, 2)))).to(dev)
    p2 = torch.from_numpy(sc.tracks[1:]).to(dev)
    valid = torch.from_numpy(sc.mask[1:]).to(dev)
    np.random.seed(0)
    smp = tv.generate_samples(N, a.trials, 7)

    def call():
        return tv.estimate_fundamental(p1, p2, max_error=a.max_error, lo_num=a.lo, valid_mask=valid, samples=smp)

    for _ in range(a.warmup):
        call()
    torch.cuda.synchronize()
    clocks = ClockSampler(dev.index or 0)
    clocks.prepare()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    clocks.start()
    e0.record()
    for _ in range(a.iters):
        out = call()
    e1.record()
    torch.cuda.synchronize()
    clk = clocks.stop()
    ms = e0.elapsed_time(e1) / a.iters

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        for k, ph in PHASES.items():
            if k in ev.key:
                split[ph] = split.get(ph, 0.0) + ev.device_time_total / 1e3        # us -> ms
    nvalid = int(valid.sum())
    evals_min = 3 * a.trials * nvalid
    lo_total = a.lo + a.lo // 2
    evals_lo = 2 * lo_total * B * N
    sm_mhz = clk.get("sm_mhz")
    props = torch.cuda.get_device_properties(dev)
    bound_ms = None
    if sm_mhz:
        bound_ms = evals_min * FP64_OPS_PER_EVAL / (props.multi_processor_count * FP64_OPS_PER_CLK_PER_SM * sm_mhz * 1e6) * 1e3
    mn = split.get("minimal+scoring")
    print(json.dumps({
        "workload": f"{B} pairs x {N} matches, T={a.trials}, lo={a.lo}, threshold {a.max_error ** 2:g} px^2, "
                    f"30% invisible, 5% outliers, float32 tracks",
        "gpu": props.name, "ms_per_call": round(ms, 3),
        "sampson_evals_per_call": {"minimal": evals_min, "lo": evals_lo},
        "sampson_evals_per_s": (evals_min + evals_lo) / (ms * 1e-3),
        "kernel_ms": {k: round(v, 3) for k, v in split.items()},
        "minimal_fp64_bound_ms": None if bound_ms is None else round(bound_ms, 3),
        "minimal_share_of_fp64_bound": None if (bound_ms is None or not mn) else round(bound_ms / mn, 3),
        "clocks": clk, "inliers_pair0": int(out[1][0]),
    }))


def _card(index):
    """(name, enforced power limit in W) through NVML, or (name, None)."""
    import torch
    name = torch.cuda.get_device_properties(index).name
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        return name, pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        return name, None


def bench_poselib(a):
    import ctypes
    import time
    import torch
    from bench import ClockSampler
    from oracle import poselib_oracle as po
    from vggsfm_b200 import _lib
    from vggsfm_b200 import two_view as tv
    from vggsfm_b200.synthetic import make_scene
    if not torch.cuda.is_available():
        raise SystemExit("twoview_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    B, N, min_it = a.pairs, a.points, 1000
    sc = make_scene(B + 1, N, seed=0, invisible_frac=0.3, outlier_frac=0.05)
    p1 = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(sc.tracks[:1], (B, N, 2)))).to(dev)
    p2 = torch.from_numpy(sc.tracks[1:]).to(dev)
    valid = torch.from_numpy(sc.mask[1:]).to(dev)
    nb = ctypes.c_size_t()
    _lib.check(_lib.lib().vgg_msac_fundamental_workspace_bytes(B, N, a.max_iterations, min_it, ctypes.byref(nb)), "ws")
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)

    def call():
        return tv.estimate_fundamental_msac(p1, p2, valid, max_error=a.max_error, max_iterations=a.max_iterations,
                                            min_iterations=min_it, workspace=ws)

    for _ in range(a.warmup):
        call()
    torch.cuda.synchronize()
    card, power_w = _card(dev.index or 0)
    clocks = ClockSampler(dev.index or 0)
    clocks.prepare()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    clocks.start()
    e0.record()
    for _ in range(a.iters):
        out = call()
    e1.record()
    torch.cuda.synchronize()
    clk = clocks.stop()
    ms = e0.elapsed_time(e1) / a.iters
    runs = np.zeros(B, np.int32)
    win = np.zeros(B, np.int32)
    trials = np.zeros((B, 1), np.int32)
    _lib.check(_lib.lib().vgg_dev_msac_trace(B, N, a.max_iterations, min_it, ws.data_ptr(), 1, runs.ctypes.data,
                                             win.ctypes.data, trials.ctypes.data), "trace")
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        m = re.search(r"\bms_[a-z_]+_kernel", ev.key)
        if m:
            split[m.group(0)] = split.get(m.group(0), 0.0) + ev.device_time_total / 1e3
    iters = out[3].cpu().numpy()
    nval = valid.sum(1).cpu().numpy().astype(np.int64)
    # Sampson evaluations: 3 candidate slots per computed trial (whole chunks of min_iterations + 1) and about 27
    # passes per LO run (25 LM iterations, the start and the MSAC score), plus the final LO and polish
    chunks = np.ceil(iters / float(min_it + 1)) * (min_it + 1)
    evals = float((3 * np.minimum(chunks, a.max_iterations) * nval).sum() + (27 * (runs + 1) * nval).sum())
    hist = {int(k): int(v) for k, v in zip(*np.unique(iters, return_counts=True))}
    rows = list(range(min(a.oracle_pairs, B)))
    t0 = time.perf_counter()
    po.estimate_fundamental_msac(p1.cpu().numpy(), p2.cpu().numpy(), sc.mask[1:], a.max_error, a.max_iterations,
                                 min_it, pairs=rows)
    oracle_s = (time.perf_counter() - t0) / max(len(rows), 1)
    print(json.dumps({
        "workload": f"{B} pairs x {N} matches, LO-MSAC (poselib.estimate_fundamental), max_error {a.max_error:g} px, "
                    f"max_iterations {a.max_iterations}, min_iterations {min_it}, 30% invisible, 5% outliers, "
                    f"float32 tracks",
        "gpu": card, "power_limit_w": power_w, "ms_per_call": round(ms, 3),
        "iterations_histogram": hist, "lo_runs_per_pair": {"mean": float(runs.mean()), "max": int(runs.max())},
        "sampson_evals_per_call": evals, "sampson_evals_per_s": evals / (ms * 1e-3),
        "kernel_ms": {k: round(v, 3) for k, v in sorted(split.items())},
        "cpu_oracle_s_per_pair": round(oracle_s, 3), "cpu_oracle_note": "restatement, not PoseLib",
        "clocks": clk, "inliers_pair0": int(out[1][0]),
    }))


if __name__ == "__main__":
    main()
