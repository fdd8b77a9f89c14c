"""Where a Gauss-Newton iteration of the streamed solver spends its time, on bench.py's C2 workload.

Mode `phases` runs one solve pass with the GN loop kernel's cycle counters on (plstvo_batch_phase_cycles; the pass computes
what the plain pass computes) and prints, per GN stage, the cycles of each phase per iteration (median and p90 over the
problems of the batch), the iterations per stage, K2's cycles per phase over the pairs it solved, and the whole-kernel times of
the other streamed-solver kernels (CUDA events).  Mode `trace` records a torch.profiler CUDA-activity trace of a few resident passes (what bench.py times) into the
output directory and reports, per pass and stream, when each kernel started and ended, and how much of the pass is solver
time after the last matcher kernel has ended.  Both print the card, its power limit and the SM clock sampled in the run.

    python tools/probe_solver_phases.py [--mode phases|trace|both] [--out DIR] [--pairs 512] [--passes 3]

Writes only under --out (default: a new temporary directory).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["wait", "eval", "fold", "barrier", "tests", "close", "solve", "increment", "trailing", "inv6"]
PER_CALL = {"wait", "inv6"}          # once per call (the first iteration's record load, the end-of-call covariance)
GL_FIRST, GL_N = 8, 11                # include/plstvo.h, PLSTVO_PHASE_SLOTS
# K2's slots 0 .. GL_FIRST - 1, cycles per pair (sort_mad is part of outliers)
K2_PHASES = ["match_finalize", "gather", "gn_eval", "gn_serial", "gates_eig", "outliers", "final", "sort_mad"]
MATCHER = ("tc_hamming_kernel", "tc_resolve_kernel")
SOLVER = ("stream_prepare_kernel", "gn_loop_stream_kernel", "stream_outlier_kernel", "stream_finalize_kernel",
          "track_solve_kernel")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--mode", choices=["phases", "trace", "both"], default="both")
    ap.add_argument("--out", default=None, help="output directory (created; default: a new temporary directory)")
    ap.add_argument("--pairs", type=int, default=512, help="frame pairs per pass (bench.py's C2: 512)")
    ap.add_argument("--passes", type=int, default=3, help="resident passes recorded in trace mode")
    return ap.parse_args(argv)


def output_dir(out):
    d = out if out else tempfile.mkdtemp(prefix="solver_phases_")
    os.makedirs(d, exist_ok=True)
    return os.path.abspath(d)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"unavailable ({e})"


def phase_table(cyc):
    """cyc: [B][PHASE_SLOTS] -> {stage: {phase: (median, p90) cycles per iteration (per call for PER_CALL)}, iterations}"""
    out = {}
    for s in range(2):
        blk = cyc[:, GL_FIRST + s * GL_N: GL_FIRST + (s + 1) * GL_N].astype(np.float64)
        iters = blk[:, GL_N - 1]
        ran = iters > 0
        st = {"problems": int(ran.sum())}
        if ran.any():
            it = iters[ran]
            st["iterations"] = {"mean": float(it.mean()), "median": float(np.median(it)), "max": int(it.max()),
                                "histogram": {int(k): int(v) for k, v in zip(*np.unique(it, return_counts=True))}}
            total = np.zeros(int(ran.sum()))
            for k, name in enumerate(PHASES):
                v = blk[ran, k] / (1.0 if name in PER_CALL else it)
                st[name] = {"median": float(np.median(v)), "p90": float(np.percentile(v, 90))}
                total += blk[ran, k]
            per_it = total / it
            st["per_iteration_total"] = {"median": float(np.median(per_it)), "p90": float(np.percentile(per_it, 90))}
        out[f"stage{s + 1}"] = st
    return out


def k2_table(cyc):
    """cyc: [B][PHASE_SLOTS] -> {phase: (median, p90) cycles per pair} of K2 over the pairs whose K2 slots are non-zero (the pairs
    K2 solved: all of them when it is the solver, those handed back to it by the streamed solver otherwise)"""
    blk = cyc[:, :len(K2_PHASES)].astype(np.float64)
    ran = (blk != 0).any(axis=1)
    tab = {"pairs": int(ran.sum())}
    if ran.any():
        for k, name in enumerate(K2_PHASES):
            tab[name] = {"median": float(np.median(blk[ran, k])), "p90": float(np.percentile(blk[ran, k], 90))}
    return tab


def print_k2_table(tab, mhz):
    if not tab["pairs"]:
        print("K2: no pair ran")
        return
    print(f"K2: {tab['pairs']} pairs")
    print(f"  {'phase':<20}{'median':>10}{'p90':>10}   cycles per pair" + (f" (us at {mhz:.0f} MHz)" if mhz else ""))
    for name in K2_PHASES:
        v = tab[name]
        us = f"  {v['median'] / mhz:7.2f} us" if mhz else ""
        print(f"  {name:<20}{v['median']:>10.0f}{v['p90']:>10.0f}{us}")


def print_table(tab, mhz):
    for s, st in tab.items():
        if "iterations" not in st:
            print(f"{s}: no problem ran")
            continue
        i = st["iterations"]
        print(f"{s}: {st['problems']} problems, iterations mean {i['mean']:.2f} median {i['median']:.0f} max {i['max']} "
              f"histogram {i['histogram']}")
        print(f"  {'phase':<20}{'median':>10}{'p90':>10}   cycles" + (f" (us at {mhz:.0f} MHz)" if mhz else ""))
        for name in PHASES + ["per_iteration_total"]:
            v = st[name]
            unit = "per call" if name in PER_CALL else "per iteration"
            us = f"  {v['median'] / mhz:7.2f} us" if mhz else ""
            print(f"  {name:<20}{v['median']:>10.0f}{v['p90']:>10.0f}   {unit}{us}")


def run_phases(db, eng, out):
    from bench import ClockSampler
    with ClockSampler(0) as clk:
        for _ in range(3):
            db.run()
        eng.synchronize()
        cyc = db.phase_cycles()
        st = db.stage_times(iters=5)
    clocks = clk.summary()
    np.save(os.path.join(out, "phase_cycles.npy"), cyc)
    tab = phase_table(cyc)
    k2 = k2_table(cyc)
    kernels = {"stream_prepare_kernel": st["ms_lists"], "gn_loop_stream_kernel stage 1": st["ms_gn_stage1"],
               "stream_outlier_kernel": st["ms_outliers"], "gn_loop_stream_kernel stage 2": st["ms_gn_stage2"],
               "stream_finalize_kernel + handed-back problems":
                   max(st["ms_optimize_pose"] - st["ms_gn_stage1"] - st["ms_gn_stage2"] - st["ms_outliers"], 0.0)}
    print_table(tab, clocks.get("sm_mhz"))
    print_k2_table(k2, clocks.get("sm_mhz"))
    print("whole kernels (ms, CUDA events, each stage alone over the batch):")
    for k, v in kernels.items():
        print(f"  {k:<48}{v:8.4f}")
    return {"phases": tab, "k2_phases": k2, "kernels_ms": kernels, "clocks": clocks}


def trace_kernels(path):
    ev = json.load(open(path))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    ks = [e for e in ev if e.get("cat") == "kernel" and e.get("ph") == "X"]
    return sorted(({"name": e["name"], "stream": e.get("args", {}).get("stream"), "ts": float(e["ts"]),
                    "end": float(e["ts"]) + float(e["dur"])} for e in ks), key=lambda k: k["ts"])


def short(name):
    for k in MATCHER + SOLVER:
        if k in name:
            return k
    return name.split("(")[0][-48:]


def split_passes(ks, gap_us=500.0):
    passes, cur, end = [], [], None
    for k in ks:
        if cur and k["ts"] - end > gap_us:
            passes.append(cur)
            cur, end = [], None
        cur.append(k)
        end = k["end"] if end is None else max(end, k["end"])
    if cur:
        passes.append(cur)
    return passes


def union_after(intervals, t0):
    iv = sorted((max(a, t0), b) for a, b in intervals if b > t0)
    tot, cur_a, cur_b = 0.0, None, None
    for a, b in iv:
        if cur_b is None or a > cur_b:
            if cur_b is not None:
                tot += cur_b - cur_a
            cur_a, cur_b = a, b
        else:
            cur_b = max(cur_b, b)
    return tot + ((cur_b - cur_a) if cur_b is not None else 0.0)


def pass_report(ks):
    t0 = ks[0]["ts"]
    span = max(k["end"] for k in ks) - t0
    m_end = max((k["end"] for k in ks if short(k["name"]) in MATCHER), default=t0)
    solver = [(k["ts"], k["end"]) for k in ks if short(k["name"]) in SOLVER]
    gn_first = min((k["ts"] for k in ks if short(k["name"]) == "gn_loop_stream_kernel"), default=None)
    after = union_after(solver, m_end)
    streams = {}
    for k in ks:
        streams.setdefault(str(k["stream"]), []).append(
            {"kernel": short(k["name"]), "start_us": round(k["ts"] - t0, 2), "end_us": round(k["end"] - t0, 2)})
    return {"span_us": span, "last_matcher_end_us": m_end - t0, "solver_after_matcher_us": after,
            "solver_after_matcher_share": after / span if span > 0 else 0.0,
            "first_gn_start_us": None if gn_first is None else gn_first - t0,
            "gn_starts_after_last_matcher": gn_first is not None and gn_first >= m_end, "streams": streams}


def run_trace(db, eng, out, passes):
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        db.run()
    eng.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(passes):
            db.run()
            eng.synchronize()
            time.sleep(0.005)          # a host gap between passes: the trace is split at it
    torch.cuda.synchronize()
    path = os.path.join(out, "resident_passes.pt.trace.json")
    prof.export_chrome_trace(path)
    reps = [pass_report(p) for p in split_passes(trace_kernels(path))]
    for i, r in enumerate(reps):
        print(f"pass {i}: span {r['span_us']:.1f} us, last matcher kernel ends at {r['last_matcher_end_us']:.1f} us, "
              f"first GN loop starts at {r['first_gn_start_us']} us, solver time after it {r['solver_after_matcher_us']:.1f} us "
              f"({100 * r['solver_after_matcher_share']:.1f} % of the pass)")
        for s, lst in r["streams"].items():
            print(f"  stream {s}: " + ", ".join(f"{k['kernel']} {k['start_us']:.1f}-{k['end_us']:.1f}" for k in lst))
    return {"trace": path, "passes": reps}


def main(argv=None):
    args = parse_args(argv)
    out = output_dir(args.out)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("probe_solver_phases: no CUDA device (the probe measures on the GPU and has no CPU path)")
    from bench import make_workload, workload_config
    from stvo_pl_b200.engine import Engine
    eng = Engine(0)
    prev, curr, _, cam = make_workload(args.pairs, 0)
    db = eng.upload(cam, workload_config(), prev, curr)
    rep = {"card": card(), "pairs": args.pairs, "out": out}
    print(f"card: {rep['card']}")
    if args.mode in ("phases", "both"):
        rep.update(run_phases(db, eng, out))
    if args.mode in ("trace", "both"):
        rep.update(run_trace(db, eng, out, args.passes))
    with open(os.path.join(out, "solver_phases.json"), "w") as f:
        json.dump(rep, f, indent=1)
    print(f"written: {out}")
    db.free()
    eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
