"""What drawing each new frame's plotStereoFrame image on the device costs, against the host path a viewer takes without it.
plstvo_stereo_session_insert on colour frames through a colour rectifier with KITTI's cam_d0 maps, timed three ways in one
process on one context, the arms alternating frame by frame: retention on without plotting; retention and plotting on,
followed by plstvo_stereo_session_read_plot; and, where cv2 imports, retention on followed by plstvo_stereo_session_read,
cv2.remap of each colour left image and cv2.circle / cv2.line of the read rows on one host thread.  KITTI-size moving views
(1241x376, BGR), the shipped ORB (1200 features, 4 levels) and LSD options, two workloads: 1 stream x 50 frames, and
sm_count + 5 streams x 8 rounds.  The arms' results and n_stereo are compared byte for byte, and the host images with
read_plot's.  Prints one JSON line per workload: each arm's wall time per call (median, min, max; a session call returns
synchronised), read_plot's time and bytes, the plot arena's device bytes, and the card's name and power limit read in the
same run.

    python tools/bench_session_plot.py --gpus 1
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

from bench_session_frames import stats  # noqa: E402
from bench_stereo_session import W, H, card, frames, scenes  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402


def colour_scenes(sc):
    """BGR frames whose channels differ, from the grey scenes"""
    from test_gpu_session_cams import colour
    return [colour(d, s) for s, d in enumerate(sc)]


def host_plot(cv2, img_l, maps, pt, ls):
    """the viewer's host path: cv2.remap of each colour left image, then plotStereoFrame's draws of the read rows"""
    out = []
    po = np.concatenate([[0], np.cumsum(pt["counts"])])
    lo = np.concatenate([[0], np.cumsum(ls["counts"])])
    for k in range(len(img_l)):
        img = cv2.remap(img_l[k], maps[0], maps[1], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        for x, y in pt["pl"][po[k]:po[k + 1]]:
            cv2.circle(img, (int(x), int(y)), 3, (0, 200, 0), 1)
        for s, e in zip(ls["spl"][lo[k]:lo[k + 1]], ls["epl"][lo[k]:lo[k + 1]]):
            cv2.line(img, (int(s[0]), int(s[1])), (int(e[0]), int(e[1])), (0, 200, 0), 1)
        out.append(img)
    return np.stack(out)


def run(e, cam, cfgs, rect, maps, cv2, sc_frames, S, steps):
    """One workload: S streams, `steps` inserts after one initialize; returns its JSON record."""
    tc, mc, sc, oc, lc = cfgs
    ids = np.arange(S, dtype=np.int32)
    names = ["retain", "plot"] + (["host"] if cv2 is not None else [])
    arms = {name: e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, S) for name in names}
    for ss in arms.values():
        ss.retain(True)
    arms["plot"].plot(True)
    for ss in arms.values():
        ss.initialize(ids, frames(sc_frames, S, 0, 20))
    t = {name: [] for name in arms}
    t_read, read_bytes = [], 0
    for k in range(1, steps + 1):
        curr = frames(sc_frames, S, k, 20)
        order = names[k % len(names):] + names[:k % len(names)]   # rotate the order: no arm always runs first
        got, imgs = {}, {}
        for name in order:
            t0 = time.perf_counter()
            got[name] = arms[name].insert(ids, curr)
            t1 = time.perf_counter()
            if name == "plot":
                imgs[name] = arms[name].read_plot()
                t2 = time.perf_counter()
                t_read.append((t2 - t1) * 1e3)
                read_bytes = imgs[name].nbytes
            elif name == "host":
                pt, ls = arms[name].read()[:2]
                imgs[name] = host_plot(cv2, curr["img_l"], maps, pt, ls)
                t2 = time.perf_counter()
            else:
                t2 = t1
            t[name].append((t2 - t0) * 1e3)
        for name in names[1:]:
            if any(x.tobytes() != y.tobytes() for x, y in zip(got[name], got["retain"])):
                raise SystemExit(f"S={S} step {k}: arm {name} differs from retention alone")
        if "host" in imgs and not np.array_equal(imgs["host"], imgs["plot"]):
            raise SystemExit(f"S={S} step {k}: read_plot's images differ from the host path's")
    rec = dict(streams=S, inserts=steps, identical=True, host_arm=cv2 is not None,
               call_ms={name: stats(v) for name, v in t.items()},
               read_plot_ms=stats(t_read), read_plot_bytes_last=int(read_bytes),
               device_bytes=dict(retain=arms["retain"].device_bytes, plot=arms["plot"].device_bytes,
                                 plot_arena=arms["plot"].device_bytes - arms["retain"].device_bytes))
    for ss in arms.values():
        e.stereo_session_destroy(ss)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1: a session lives on one device")
    ap.add_argument("--frames", type=int, default=50, help="inserts of the one-stream workload")
    ap.add_argument("--rounds", type=int, default=8, help="inserts of the many-stream workload")
    ap.add_argument("--scenes", type=int, default=16)
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("--gpus 1 only")
    try:
        import cv2
        cv2.setNumThreads(1)   # the viewer's one host thread
    except ImportError:
        cv2 = None
    from test_gpu_rectify import rig
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    cfgs = (tc, mc, sc, oc, lc)
    cam, m = rig("kitti")
    maps = m[:2]
    name, power = card()
    e = Engine()
    rect = e.rectifier_create_color(W, H, 3, *m)
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # warm-up (not timed): every arena of a 1-stream and an S-stream call
    warm = colour_scenes(scenes(2, 2))
    run(e, cam, cfgs, rect, maps, cv2, warm, 1, 1)
    run(e, cam, cfgs, rect, maps, cv2, warm, sms + 5, 1)
    for S, steps, n_scenes in ((1, a.frames, 1), (sms + 5, a.rounds, a.scenes)):
        rec = run(e, cam, cfgs, rect, maps, cv2, colour_scenes(scenes(n_scenes, steps + 1)), S, steps)
        print(json.dumps(dict(card=name, power_limit=power, width=W, height=H, **rec)), flush=True)
    e.rectifier_destroy(rect)
    e.close()


if __name__ == "__main__":
    main()
