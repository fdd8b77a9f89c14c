"""What a stereo session costs on the reference's FLD line branch (plstvo_stereo_session_use_fld_lines), where the caller
brings each frame's key lines and LSD does not run, against the same session running LSD.  LSD's own key lines, computed
once per scene frame before any timed region (plstvo_lsd_detect_batch), stand in for FastLineDetector's, so on grey frames
the two sessions must give the same bytes; every rep checks that (results, n_stereo, threshold rows), and that each
session's run equals its per-frame loop.  Arms, alternating in order rep by rep on twin sessions initialised from the same
frames: the per-frame insert loop (the FAST threshold and prior carried on the host, handler.update_fast_threshold) and one
run of T steps, each with the switch on and off.  Prints one JSON line per workload: wall ms per frame (T S frames; median,
min, max over the reps; every arm returns synchronised), the FLD run's stage times (plstvo_track_stereo_images_stage_times),
each run session's device memory after its run (plstvo_stereo_session_device_bytes: the session's pools), the device memory
one run takes in all (the run alone in a fresh context: cudaMemGetInfo before the context is created and after the run, so
the context's arenas, LSD's included, and the session), and the card's name and power limit read in the same process.
  KITTI size (1241x376) moving grey views, shipped ORB (1200 features, 4 levels) and LSD options, KITTI handler config;
  S in {1, 8, 64} streams, T in {8, 32} frames.  An LSD arm whose images would need more device memory than --max-gb
  (LSD's 35 bytes or so per scaled pixel) is reported as not run; the FLD arms keep no LSD arena and run.
  BGR rows: EuRoC size (752x480) BGR frames through a colour rectifier with maps (the rig the tests use), the same S and
  T; there LBD reads the RGB2GRAY plane, so the FLD session is checked against its own loop only.

    python tools/bench_session_fld.py --gpus 1
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_session_run import colour, loop, stats, views  # noqa: E402
from bench_stereo_session import card  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402
from stvo_pl_b200.handler import HandlerConfig  # noqa: E402


def scene_lines(e, lc, st, rect):
    """lines[s][f] = ((seg, angle, npix) left, right) of scene s's frame f, on the grey image the session's stages see"""
    out = []
    for d in st:
        il, ir = d["img_l"], d["img_r"]
        if rect is not None:
            il, ir = e.rectify_batch(rect, il, ir)
        n = len(il)
        _, kl = e.lsd_detect_batch(lc, np.concatenate([il, ir]))
        o = kl["off"]
        cut = lambda i: tuple(kl[k][o[i]:o[i + 1]] for k in ("seg", "angle", "npix"))  # noqa: E731
        out.append([(cut(f), cut(n + f)) for f in range(n)])
    return out


def fields(lines, keys):
    """the key-line fields of frames keys [(scene, frame)], frame-major"""
    d = {}
    for side, o, sg, an, npx in ((0, "ll_off", "seg_l", "angle_l", "npix_l"), (1, "lr_off", "seg_r", "angle_r", "npix_r")):
        parts = [lines[s][f][side] for s, f in keys]
        d[o] = np.concatenate([[0], np.cumsum([len(p[2]) for p in parts])]).astype(np.int32)
        d[sg] = np.concatenate([p[0] for p in parts]).reshape(-1, 4)
        d[an] = np.concatenate([p[1] for p in parts])
        d[npx] = np.concatenate([p[2] for p in parts])
    return d


def fld_loop(ss, h, th0, ids, frames, T_, lines_of):
    """bench_session_run.loop with each step's key lines"""
    class Wrap:
        def insert(self, ids_, fr, pri):
            t = Wrap.t
            Wrap.t += 1
            return ss.insert(ids_, dict(fr, **lines_of(t)), pri)
    Wrap.t = 0
    return loop(Wrap(), h, th0, ids, frames, T_)


def run_bytes(cfgs, cam, rect_args, S, T_, fld, h, ids, th0, init, frames):
    """device memory one run takes in a fresh context: cudaMemGetInfo before the context exists and after the run"""
    import torch
    tc, mc, sc, oc, lc = cfgs
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    e2 = Engine()
    rect = None if rect_args is None else e2.rectifier_create_color(*rect_args)
    ss = e2.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, S)
    if fld:
        ss.use_fld_lines(True)
    ss.initialize(ids, init)
    ss.run(h, ids, T_, frames, th0)
    used = free0 - torch.cuda.mem_get_info()[0]
    e2.close()
    return int(used)


def workload(e, cfgs, cam, rect, st, lines, S, T_, reps, lsd_fits, rect_args=None):
    tc, mc, sc, oc, lc = cfgs
    h = HandlerConfig(fast_min_th=7, fast_max_th=30)   # config_kitti.yaml
    ids = np.arange(S, dtype=np.int32)
    th0 = np.full(S, 20, np.int32)
    names = ["fld_run", "fld_loop"] + (["lsd_run", "lsd_loop"] if lsd_fits else [])
    ss = {k: e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, S) for k in names}
    for k in names:
        if k.startswith("fld"):
            ss[k].use_fld_lines(True)
    n_sc = len(st)
    init = {k: np.stack([st[s % n_sc][k][0] for s in range(S)]) for k in ("img_l", "img_r")}
    init_lines = fields(lines, [(s % n_sc, 0) for s in range(S)])
    frames = {k: np.concatenate([np.stack([st[s % n_sc][k][t] for s in range(S)]) for t in range(1, T_ + 1)])
              for k in ("img_l", "img_r")}
    run_lines = fields(lines, [(s % n_sc, t) for t in range(1, T_ + 1) for s in range(S)])
    step_lines = [fields(lines, [(s % n_sc, t) for s in range(S)]) for t in range(1, T_ + 1)]
    times = {k: [] for k in names}
    stage, dev = [], {}
    for r in range(reps):
        for k in names:
            ss[k].initialize(ids, dict(init, **init_lines) if k.startswith("fld") else init)
        arms = {"fld_run": lambda: ss["fld_run"].run(h, ids, T_, dict(frames, **run_lines), th0),
                "fld_loop": lambda: fld_loop(ss["fld_loop"], h, th0, ids, frames, T_, lambda t: step_lines[t]),
                "lsd_run": lambda: ss["lsd_run"].run(h, ids, T_, frames, th0),
                "lsd_loop": lambda: loop(ss["lsd_loop"], h, th0, ids, frames, T_)}
        order = names[r % len(names):] + names[:r % len(names)]
        out = {}
        for k in order:
            t0 = time.perf_counter()
            out[k] = arms[k]()
            times[k].append((time.perf_counter() - t0) * 1e3 / (S * T_))
            if k == "fld_run":
                stage.append(e.track_stereo_images_stage_times().tolist())
            if k.endswith("run"):
                dev[k] = ss[k].device_bytes
        same = lambda a, b: a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])  # noqa: E731
        pairs = [("fld_run", "fld_loop")] + ([("lsd_run", "lsd_loop")] if lsd_fits else [])
        if lsd_fits and rect is None:
            pairs.append(("fld_run", "lsd_run"))
        for a, b in pairs:
            if not same(out[a], out[b]):
                raise SystemExit(f"S={S} T={T_} rep {r}: {a} and {b} differ")
    for s in ss.values():
        s.close()
    run_total = {"fld_run": run_bytes(cfgs, cam, rect_args, S, T_, True, h, ids, th0, dict(init, **init_lines),
                                      dict(frames, **run_lines))}
    if lsd_fits:
        run_total["lsd_run"] = run_bytes(cfgs, cam, rect_args, S, T_, False, h, ids, th0, init, frames)
    res = dict(S=S, T=T_, width=cam.width, height=cam.height, colour=rect is not None, byte_identical=True,
               fld_run_stage_ms_median=[float(np.median([s[k] for s in stage])) for k in range(5)],
               run_session_device_bytes={k: int(v) for k, v in dev.items()},
               run_device_bytes_fresh_context=run_total, reps=reps)
    for k in names:
        res[k + "_ms_per_frame"] = stats(times[k])
    if not lsd_fits:
        res["lsd_arms"] = "not run: LSD's resident images exceed --max-gb"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1,8,64")
    ap.add_argument("--steps", default="8,32")
    ap.add_argument("--max-gb", type=float, default=60.0, help="largest estimated LSD image residency an LSD arm may take")
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("--gpus 1 only")
    if a.reps < 3:
        raise SystemExit("--reps must be at least 3")
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    oc.fast_threshold = 0   # as the handlers set it: every frame at the handler's threshold
    cfgs = (tc, mc, sc, oc, lc)
    name, power = card()
    head = dict(card=name, power_limit=power)
    e = Engine()
    cam = T.kitti_camera()
    sizes, steps = [int(x) for x in a.sizes.split(",")], [int(x) for x in a.steps.split(",")]
    st = views(8, max(steps) + 1, cam.width, cam.height, 5100)   # stream s views scene s % 8
    lines = scene_lines(e, lc, st, None)
    workload(e, cfgs, cam, None, st, lines, 2, 2, 3, True)   # warm-up, not reported

    def fits(c, S, T_):
        scaled_px = round(c.width * lc.scale) * round(c.height * lc.scale)
        return 2 * S * T_ * scaled_px * 35 / 1e9 <= a.max_gb

    for S in sizes:
        for T_ in steps:
            print(json.dumps(dict(head, **workload(e, cfgs, cam, None, st, lines, S, T_, a.reps, fits(cam, S, T_)))), flush=True)
    from test_gpu_rectify import rig
    ecam, maps = rig("euroc")
    rect_args = (ecam.width, ecam.height, 3, *maps)
    rect = e.rectifier_create_color(*rect_args)
    est = colour(views(8, max(steps) + 1, ecam.width, ecam.height, 5300))
    elines = scene_lines(e, lc, est, rect)
    for S in sizes:
        for T_ in steps:
            print(json.dumps(dict(head, **workload(e, cfgs, ecam, rect, est, elines, S, T_, a.reps, fits(ecam, S, T_),
                                                   rect_args))), flush=True)
    e.close()


if __name__ == "__main__":
    main()
