"""Batches with more pairs than the GPU has SMs, against the oracle: what the benchmark measures.

At that size the host code cuts a batch into chunks (capi.cu: chunk_schedule for plstvo_track_batch, pass_chunk for the resident
pass and plstvo_track_batch_async), each chunk with its own pair offset, feature-scratch slice, queue words, matcher item range,
uploads and downloads, on two alternating compute streams; the default policy picks the streamed solver; and the streamed solver's
persistent CTAs (2 per SM) each take several problems from the queue, carrying the TMA ring's phases from one problem to the
next.  None of that happens at B <= sm_count.  PLSTVO_STREAM_SOLVE / PLSTVO_K2_FEAT_GLOBAL are read once per process, so runs that
pin them go through a subprocess (inputs and outputs pickled / saved in a temporary directory); the oracle runs in this process."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import ref_numpy as R
from stvo_pl_b200 import synth, types as T
from test_gpu_pose import TOL_ANG, TOL_TR, compare

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# what the streamed solver reaches on a C2 pair (2500 matched features) whose inlier flags all equal the oracle's; its fp32
# evaluation noise on the solution grows as 1 / sqrt(n) on shorter lists (measured: 1.4e-6 m on a pair of 268 matches whose stage 2
# ran into max_iters_ref), so the bar is scaled by sqrt(2500 / n) below that length
STREAM_ANG, STREAM_TR, STREAM_N = 1e-7, 1e-6, 2500
GS_PT_TILE, GS_LS_TILE, GL_STAGES = 512, 256, 6   # record tiles and ring stages of gn_loop_stream_kernel (gn_stream.cuh, solve.cu)


# ---- mirror of capi.cu's chunking: only used to place special pairs on chunk bounds and to check a batch spans several chunks ----
def pass_chunk(B, sm_count):
    return max(1, max(min(B, sm_count), (B + 1) // 2))


def chunk_schedule(B, sm_count, pipelined):
    if pipelined:
        return list(range(0, B, pass_chunk(B, sm_count))) + [B]
    bounds, p, c = [0], 0, max(8, sm_count // 6)
    while c < sm_count and p + c < B:
        p += c
        bounds.append(p)
        c *= 2
    rest = B - p
    if rest > 0:
        n = (rest + sm_count - 1) // sm_count
        bounds += [p + rest * k // n for k in range(1, n + 1)]
    return bounds


def test_chunk_schedule_mirror_examples():
    """The bounds the H100 (132 SMs) takes at the benchmark's batch size."""
    assert chunk_schedule(512, 132, False) == [0, 22, 66, 154, 273, 392, 512]
    assert chunk_schedule(512, 132, True) == [0, 256, 512]
    assert chunk_schedule(22, 132, False) == [0, 22] and chunk_schedule(23, 132, False) == [0, 22, 23]
    assert chunk_schedule(132, 132, True) == [0, 132] and chunk_schedule(133, 132, True) == [0, 132, 133]


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _threads():
    return os.cpu_count() or 1


# ---- subprocess runner: a list of calls on one Engine under a given environment ----
SCRIPT = r'''
import json, pickle, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from stvo_pl_b200.engine import Engine
job = pickle.load(open(sys.argv[2], "rb"))
eng = Engine(0)
out = {}
for k, call in enumerate(job["calls"]):
    if call[0] == "track":
        _, cam, cfg, prev, curr, pri = call
        g = eng.track_batch(cam, cfg, prev, curr, priors=pri)
        for key, v in g.items():
            out["%d_%s" % (k, key)] = v
        if k == 0:   # which solver form the policy chose for the whole batch, and what it handed back to K2
            db = eng.upload(cam, cfg, prev, curr, priors=pri)
            st = db.stage_times(1)
            db.free()
            out["stage"] = np.array(json.dumps(st))
    else:
        _, cam, cfg, mb = call
        res, ip, il = eng.optimize_pose(cam, cfg, mb)
        out["%d_results" % k], out["%d_inlier_pt" % k], out["%d_inlier_ls" % k] = res, ip, il
eng.close()
np.savez(sys.argv[3], **out)
'''


def _run_isolated(tmp_path, name, env_set, calls):
    env = {k: v for k, v in os.environ.items() if k not in ("PLSTVO_STREAM_SOLVE", "PLSTVO_K2_FEAT_GLOBAL")}
    env.update(env_set)
    job, res = os.path.join(str(tmp_path), name + ".pkl"), os.path.join(str(tmp_path), name + ".npz")
    with open(job, "wb") as f:
        pickle.dump(dict(calls=calls), f)
    r = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, job, res], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    with np.load(res) as z:
        out = {k: z[k] for k in z.files}
    os.remove(job)
    os.remove(res)
    groups = {}
    for key, v in out.items():
        if key == "stage":
            continue
        k, field = key.split("_", 1)
        groups.setdefault(int(k), {})[field] = v
    stage = json.loads(str(out["stage"])) if "stage" in out else None
    return [groups[k] for k in range(len(calls))], stage


# ---- comparisons ----
def _per_pair_flips(gpu, ref, pt_off, ls_off):
    cp = np.concatenate([[0], np.cumsum(gpu["inlier_pt"] != ref["inlier_pt"])])
    cl = np.concatenate([[0], np.cumsum(gpu["inlier_ls"] != ref["inlier_ls"])])
    return (cp[pt_off[1:]] - cp[pt_off[:-1]]) + (cl[ls_off[1:]] - cl[ls_off[:-1]])


def _check_streamed(gpu, ref, prev, label):
    """Streamed-solver bars: matching bit-exact, same branch of optimizePose per pair, pose within north_star, 1e-7 rad / 1e-6 m
    where the pair's inlier flags all equal the oracle's, and at most max(2, n // 1000) differing flags over the batch."""
    np.testing.assert_array_equal(gpu["m12_pt"], ref["m12_pt"])
    np.testing.assert_array_equal(gpu["m12_ls"], ref["m12_ls"])
    flips = _per_pair_flips(gpu, ref, prev.pt_off, prev.ls_off)
    worst, worst_clean = (0.0, 0.0), (0.0, 0.0)
    for p in range(prev.B):
        g, r = gpu["results"][p], ref["results"][p]
        assert g["status"] == r["status"] and g["good"] == r["good"], (label, p, g["status"], r["status"])
        assert g["n_matched_pt"] == r["n_matched_pt"] and g["n_matched_ls"] == r["n_matched_ls"], (label, p)
        ang, tr = R.pose_error(g["DT"], r["DT"])
        worst = (max(worst[0], ang), max(worst[1], tr))
        assert ang < TOL_ANG and tr < TOL_TR, (label, p, ang, tr)
        assert np.abs(g["Tfw"] - r["Tfw"]).max() < TOL_TR, (label, p)
        if flips[p] == 0:
            worst_clean = (max(worst_clean[0], ang), max(worst_clean[1], tr))
            scale = np.sqrt(STREAM_N / max(STREAM_N / 100, min(STREAM_N, int(r["n_matched_pt"]) + int(r["n_matched_ls"]))))
            assert ang < STREAM_ANG * scale and tr < STREAM_TR * scale, (label, p, ang, tr, scale)
    n = prev.n_pt + prev.n_ls
    print(f"{label}: worst pose deviation {worst[0]:.2e} rad / {worst[1]:.2e} m ({worst_clean[0]:.2e} / {worst_clean[1]:.2e} "
          f"on pairs without a flipped flag); {int(flips.sum())} of {n} inlier flags differ, in {int((flips > 0).sum())} pairs")
    assert flips.sum() <= max(2, n // 1000), label
    return worst


def _same_bytes(a, b, label):
    assert a["results"].tobytes() == b["results"].tobytes(), label
    for k in ("m12_pt", "m12_ls", "inlier_pt", "inlier_ls"):
        if k in a and k in b:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{label}: {k}")


def _pair_slice(out, prev, p):
    """Pair p's bytes of a track output."""
    a, b, c, d = prev.pt_off[p], prev.pt_off[p + 1], prev.ls_off[p], prev.ls_off[p + 1]
    return (out["results"][p].tobytes(), out["m12_pt"][a:b].tobytes(), out["m12_ls"][c:d].tobytes(),
            out["inlier_pt"][a:b].tobytes(), out["inlier_ls"][c:d].tobytes())


def _groups(B, bound_pairs, run=7):
    return [list(range(i, min(i + run, B))) for i in range(0, B, run)] + [[p] for p in sorted(bound_pairs)]


def _check_sub_batches(big, subs, groups, prev, label):
    """Every pair's results, m12 and inlier flags from the big batch equal those from a small batch holding the pair."""
    n = 0
    for grp, out in zip(groups, subs):
        sub_prev = prev.select(grp)
        for j, p in enumerate(grp):
            assert _pair_slice(big, prev, p) == _pair_slice(out, sub_prev, j), (label, p, grp)
            n += 1
    print(f"{label}: {n} pair solves in {len(groups)} sub-batches equal the big batch byte for byte")


# ---- 1. the benchmark's batch through every track entry point ----
@pytest.fixture(scope="module")
def c2_batch(oracle):
    cfg = T.kitti_config()
    prev, curr, _, cam = synth.make_batch("kitti", 512, overlap=1.0)
    ref = oracle.track_batch(cam, cfg, prev, curr, threads=_threads())
    return cfg, prev, curr, cam, ref


def test_bench_batch_every_entry_point_vs_oracle(engine, c2_batch, sm_count):
    cfg, prev, curr, cam, ref = c2_batch
    B = prev.B
    blocking, pipelined = chunk_schedule(B, sm_count, False), chunk_schedule(B, sm_count, True)
    assert B > sm_count and len(blocking) > 3 and len(pipelined) > 2, (sm_count, blocking, pipelined)
    print(f"B = {B}, {sm_count} SMs: plstvo_track_batch chunks {blocking}; resident / async chunks {pipelined}")

    blk = engine.track_batch(cam, cfg, prev, curr)
    _check_streamed(blk, ref, prev, "plstvo_track_batch")

    pp, pc = engine.pinned.pin_frames(prev), engine.pinned.pin_frames(curr)
    outs = [engine.pinned_outputs(prev) for _ in range(2)]
    t0 = engine.track_batch_async(cam, cfg, pp, pc, outs[0])
    t1 = engine.track_batch_async(cam, cfg, pp, pc, outs[1])     # two batches in flight, one per workspace slot
    engine.wait(t0)
    engine.wait(t1)

    db = engine.upload(cam, cfg, prev, curr)
    try:
        db.run()
        res = db.download()
        st = db.stage_times(1)
    finally:
        db.free()
    print(f"resident pass: streamed solver {st['streamed_solver']}, {st['delegated_to_fp64']} problems delegated to fp64")
    assert st["streamed_solver"], st
    # no problem of this batch is robust, falls back or stops on an increment within GL_INC_BAND of its threshold
    assert st["delegated_to_fp64"] == 0, st
    for k, out in enumerate(outs):
        _same_bytes(out, blk, f"async batch {k} vs blocking")
    _same_bytes(res, blk, "upload / run / download vs blocking")


# ---- 2. ragged batch with priors, past one wave, under each solver form ----
def _empty_like(side):
    return {k: v[:0] for k, v in side.items()}


@pytest.fixture(scope="module")
def ragged(oracle, sm_count):
    """About 2 * sm_count + 37 KITTI-size pairs of their own sizes (each side <= 2000 points + 500 lines), special pairs on the
    chunk bounds of both schedules, the first ramp chunk of plstvo_track_batch made only of pairs without a matcher problem,
    a distinct motion-model prior per pair."""
    B = 2 * sm_count + 37
    blocking, pipelined = chunk_schedule(B, sm_count, False), chunk_schedule(B, sm_count, True)
    assert len(blocking) > 4 and len(pipelined) > 2
    empty_run = range(blocking[0], blocking[1])                 # a whole chunk that launches no matcher
    bound_pairs = sorted({0, B - 1} | {q for b in blocking[1:-1] + pipelined[1:-1] for q in (b - 1, b)})
    special = [p for p in bound_pairs if p not in empty_run]
    kinds = ["curr_no_points", "curr_no_lines", "points_only", "ls_level", "few", "both_empty"]
    kind = {p: kinds[i % len(kinds)] for i, p in enumerate(special)}
    rng = np.random.default_rng(11)
    shape = synth.SHAPES["kitti"]
    prevs, currs, Ts = [], [], []
    for p in range(B):
        k = kind.get(p)
        if k == "few":
            a, c, Tg = synth.make_pair(shape, 7000 + p, n_pt=6, n_ls=2, overlap=1.0, outlier_frac=0.0)
        elif k == "both_empty" or (p in empty_run and p % 3 == 0):
            a, c, Tg = synth.make_pair(shape, 7000 + p, n_pt=0, n_ls=0)
        else:
            a, c, Tg = synth.make_pair(shape, 7000 + p, n_pt=int(rng.integers(150, 2001)),
                                       n_ls=0 if k == "points_only" else int(rng.integers(1, 501)),
                                       overlap=float(rng.uniform(0.5, 1.0)))
        if p in empty_run and p % 3 == 1:          # prev frame full, curr frame empty
            c = dict(pt=_empty_like(c["pt"]), ls=_empty_like(c["ls"]))
        elif p in empty_run and p % 3 == 2:        # prev frame points only, curr frame lines only
            a = dict(pt=a["pt"], ls=_empty_like(a["ls"]))
            c = dict(pt=_empty_like(c["pt"]), ls=c["ls"])
        elif k == "curr_no_points":
            c = dict(pt=_empty_like(c["pt"]), ls=c["ls"])
        elif k == "curr_no_lines":
            c = dict(pt=c["pt"], ls=_empty_like(c["ls"]))
        elif k == "ls_level":
            lev = (np.arange(len(a["ls"]["level"])) % 3).astype(np.int32)
            a["ls"]["level"], a["ls"]["sigma2"] = lev, 1.0 / (1.2 ** lev) ** 2
        prevs.append(a)
        currs.append(c)
        Ts.append(Tg)
    prev, curr, cam = synth._stack(prevs), synth._stack(currs), T.kitti_camera()
    pri = T.identity_priors(B)
    for p in range(B):
        pri["DT"][p] = Ts[p] @ R.expmap_se3(rng.normal(0, 0.01, 6))
        pri["DT_cov"][p] = np.eye(6) * 1e-6 * (1 + p % 5)
        pri["err_norm"][p] = 0.2
        pri["Tfw"][p] = R.expmap_se3([0.1 * p, -0.05 * p, 1.0, 0.01 * (p % 7), 0.02, -0.01 * (p % 3)])
        pri["Tfw_cov"][p] = np.eye(6) * 0.01
    cfg = T.kitti_config()
    cfg.use_motion_model = 1
    ref = oracle.track_batch(cam, cfg, prev, curr, priors=pri, threads=_threads())
    st = ref["results"]["status"]
    assert (st[[p for p in special if kind[p] == "few"]] == T.ST_FEW_BEFORE).all()
    for p in special:
        if kind[p] in ("curr_no_points", "both_empty"):
            assert (ref["m12_pt"][prev.pt_off[p]:prev.pt_off[p + 1]] == -1).all()
        if kind[p] in ("curr_no_lines", "both_empty"):
            assert (ref["m12_ls"][prev.ls_off[p]:prev.ls_off[p + 1]] == -1).all()
    print(f"ragged batch: B = {B}, plstvo_track_batch chunks {blocking}, resident / async chunks {pipelined}; "
          f"special pairs {kind}; statuses {np.bincount(st, minlength=4).tolist()}")
    return dict(cfg=cfg, cam=cam, prev=prev, curr=curr, pri=pri, ref=ref, bound_pairs=bound_pairs,
                groups=_groups(B, bound_pairs), runs={})


def _ragged_run(tmp_path, rg, setting):
    """One subprocess per solver setting, cached for the module: the big batch, then (pinned settings) every sub-batch."""
    if setting not in rg["runs"]:
        env = dict(default={}, k2=dict(PLSTVO_STREAM_SOLVE="0"), k2_global=dict(PLSTVO_STREAM_SOLVE="0", PLSTVO_K2_FEAT_GLOBAL="1"),
                   streamed=dict(PLSTVO_STREAM_SOLVE="1"))[setting]
        prev, curr, pri = rg["prev"], rg["curr"], rg["pri"]
        calls = [("track", rg["cam"], rg["cfg"], prev, curr, pri)]
        if setting != "default":
            calls += [("track", rg["cam"], rg["cfg"], prev.select(g), curr.select(g), np.ascontiguousarray(pri[g]))
                      for g in rg["groups"]]
        outs, stage = _run_isolated(tmp_path, "ragged_" + setting, env, calls)
        print(f"{setting}: streamed solver {stage['streamed_solver']}, {stage['delegated_to_fp64']} problems delegated to fp64")
        rg["runs"][setting] = (outs, stage)
    return rg["runs"][setting]


@pytest.mark.parametrize("setting", ["default", "k2", "k2_global", "streamed"])
def test_ragged_batch_with_priors_vs_oracle(tmp_path, ragged, setting):
    prev, ref = ragged["prev"], ragged["ref"]
    outs, stage = _ragged_run(tmp_path, ragged, setting)
    big = outs[0]
    if setting in ("default", "streamed"):
        assert stage["streamed_solver"], stage
        # every robust fallback (stage 1 rejected, :357-359) is handed to K2; increment hand-offs may add to them
        n_fallback = int((ref["results"]["status"] == T.ST_ROBUST_FALLBACK).sum())
        assert stage["delegated_to_fp64"] >= n_fallback, (stage, n_fallback)
        _check_streamed(big, ref, prev, f"ragged, {setting}")
    else:
        assert not stage["streamed_solver"] and stage["delegated_to_fp64"] == 0, stage
        worst = compare(big, ref, prev, tight=True, flags_exact=True)
        print(f"ragged, {setting}: K2, worst pose deviation {worst[0]:.2e} rad / {worst[1]:.2e} m, inlier flags identical")
    if setting == "k2_global":
        # the same fp64 arithmetic reading the lists from global memory instead of shared memory
        _same_bytes(big, _ragged_run(tmp_path, ragged, "k2")[0][0], "K2 global-scratch form vs shared-memory form")
    if setting == "streamed":
        _same_bytes(big, _ragged_run(tmp_path, ragged, "default")[0][0], "pinned streamed solver vs default policy")
    if setting != "default":
        _check_sub_batches(big, outs[1:], ragged["groups"], prev, f"ragged, {setting}")


# ---- 3. explicit lists: more problems than persistent CTAs, resident and streamed problems mixed ----
def _cut(mb, src, keep_pt, keep_ls):
    """Problem i = the first keep_pt[i] points / keep_ls[i] lines of problem src[i] of an equal-sized MatchedBatch."""
    ip = np.concatenate([np.arange(mb.pt_off[s], mb.pt_off[s] + k) for s, k in zip(src, keep_pt)]).astype(np.int64)
    il = np.concatenate([np.arange(mb.ls_off[s], mb.ls_off[s] + k) for s, k in zip(src, keep_ls)]).astype(np.int64)
    return T.MatchedBatch(pt_off=np.concatenate([[0], np.cumsum(keep_pt)]), ls_off=np.concatenate([[0], np.cumsum(keep_ls)]),
                          pt_P=mb.pt_P[ip], pt_pl_obs=mb.pt_pl_obs[ip], pt_sigma2=mb.pt_sigma2[ip], ls_sP=mb.ls_sP[il],
                          ls_eP=mb.ls_eP[il], ls_le_obs=mb.ls_le_obs[il], ls_spl=mb.ls_spl[il], ls_epl=mb.ls_epl[il],
                          ls_sigma2=mb.ls_sigma2[il])


def _sub_matched(mb, idx):
    ip = np.concatenate([np.arange(mb.pt_off[p], mb.pt_off[p + 1]) for p in idx]).astype(np.int64)
    il = np.concatenate([np.arange(mb.ls_off[p], mb.ls_off[p + 1]) for p in idx]).astype(np.int64)
    return T.MatchedBatch(pt_off=np.concatenate([[0], np.cumsum(np.diff(mb.pt_off)[idx])]),
                          ls_off=np.concatenate([[0], np.cumsum(np.diff(mb.ls_off)[idx])]),
                          pt_P=mb.pt_P[ip], pt_pl_obs=mb.pt_pl_obs[ip], pt_sigma2=mb.pt_sigma2[ip], ls_sP=mb.ls_sP[il],
                          ls_eP=mb.ls_eP[il], ls_le_obs=mb.ls_le_obs[il], ls_spl=mb.ls_spl[il], ls_epl=mb.ls_epl[il],
                          ls_sigma2=mb.ls_sigma2[il], pt_inlier=mb.pt_inlier[ip], ls_inlier=mb.ls_inlier[il])


# (points, lines, tiles in gn_loop_stream_kernel's ring): resident up to GL_STAGES tiles, streamed beyond
EXPLICIT_SIZES = [(400, 0, 1), (512, 256, 2), (1500, 500, 5), (2048, 512, 6), (2049, 512, 7), (8000, 2000, 24),
                  (600, 200, 3), (300, 700, 4)]


def _tiles(n, m):
    return -(-n // GS_PT_TILE) + -(-m // GS_LS_TILE)


@pytest.fixture(scope="module")
def explicit(oracle, sm_count):
    ctas = 2 * sm_count                       # gn_loop_stream_kernel's persistent grid (GL_MINBLOCKS CTAs per SM)
    B = 2 * ctas + 41
    src, _, cam = synth.make_matched_batch("hd", 16)
    rng = np.random.default_rng(5)
    cycle = len(EXPLICIT_SIZES) + 2            # + one problem with too few features, + one whose stage 1 is rejected
    keep_pt, keep_ls, kinds = [], [], []
    for i in range(B):
        j = i % cycle
        if j < len(EXPLICIT_SIZES):
            n, m, t = EXPLICIT_SIZES[j]
            assert _tiles(n, m) == t
            keep_pt.append(n); keep_ls.append(m); kinds.append(f"{t} tiles")
        elif j == len(EXPLICIT_SIZES):
            keep_pt.append(6); keep_ls.append(2); kinds.append("few")
        else:
            keep_pt.append(40); keep_ls.append(0); kinds.append("fallback")
    mb = _cut(src, [i % 16 for i in range(B)], keep_pt, keep_ls)
    # the robust-fallback construction of test_gpu_pose.test_robust_fallback_branch: 40 points on one distant spot, stage 1's
    # covariance fails isGoodSolution
    for i in range(B):
        if kinds[i] == "fallback":
            a = mb.pt_off[i]
            mb.pt_P[a:a + 40] = np.stack([rng.normal(0, 1e-4, 40), rng.normal(0, 1e-4, 40), 400 + rng.normal(0, 1e-3, 40)], 1)
            mb.pt_pl_obs[a:a + 40] = np.stack([cam.cx + rng.normal(0, 0.3, 40), cam.cy + rng.normal(0, 0.3, 40)], 1)
    # input inlier flags cleared on every third problem
    mb.pt_inlier = np.ones(len(mb.pt_sigma2), np.uint8)
    mb.ls_inlier = np.ones(len(mb.ls_sigma2), np.uint8)
    for i in range(0, B, 3):
        if kinds[i] not in ("few", "fallback"):
            a, b, c, d = mb.pt_off[i], mb.pt_off[i + 1], mb.ls_off[i], mb.ls_off[i + 1]
            mb.pt_inlier[a:b] = (np.arange(b - a) % 9 != 4)
            mb.ls_inlier[c:d] = (np.arange(d - c) % 7 != 2)
    cfg = T.kitti_config()
    rc, ref, rp, rl = oracle.optimize_pose(cam, cfg, mb)
    assert (ref["status"][[i for i in range(B) if kinds[i] == "few"]] == T.ST_FEW_BEFORE).all()
    assert (ref["status"][[i for i in range(B) if kinds[i] == "fallback"]] == T.ST_ROBUST_FALLBACK).all()
    # every CTA's queue holds more than one problem, and sees every kind
    assert B > 2 * ctas and cycle < ctas
    return dict(mb=mb, cam=cam, cfg=cfg, ref=ref, rp=rp, rl=rl, kinds=kinds, ctas=ctas)


def test_explicit_lists_past_the_persistent_grid_vs_oracle(engine, explicit, tmp_path):
    mb, cam, cfg, ref, rp, rl, kinds = (explicit[k] for k in ("mb", "cam", "cfg", "ref", "rp", "rl", "kinds"))
    B = mb.B
    res, ip, il = engine.optimize_pose(cam, cfg, mb)
    worst, n_flips = (0.0, 0.0), 0
    for p in range(B):
        assert res["status"][p] == ref["status"][p] and res["good"][p] == ref["good"][p], (p, kinds[p])
        ang, tr = R.pose_error(res["DT"][p], ref["DT"][p])
        worst = (max(worst[0], ang), max(worst[1], tr))
        assert ang < TOL_ANG and tr < TOL_TR, (p, kinds[p], ang, tr)
        a, b, c, d = mb.pt_off[p], mb.pt_off[p + 1], mb.ls_off[p], mb.ls_off[p + 1]
        flips = int((ip[a:b] != rp[a:b]).sum() + (il[c:d] != rl[c:d]).sum())
        n_flips += flips
        n = max(1, (b - a) + (d - c))
        # test_explicit_lists_c5_size's bars, scaled from its 10 000-entry lists to this list's length: a flipped flag moves the
        # error by about one feature's share (1 / n); the fp32 evaluation's noise on the error and on H averages out as
        # 1 / sqrt(n) (measured: 1.3e-6 on a 400-point list)
        err_tol = 1e-6 * np.sqrt(10000 / n) if flips == 0 else 2e-4 * flips * 10000 / n
        assert abs(res["err_norm"][p] - ref["err_norm"][p]) < err_tol, (p, kinds[p], res["err_norm"][p], ref["err_norm"][p])
        # entries far below the largest one (off-diagonal terms) carry the noise of the largest: absolute bound on the matrix's scale
        tol = 2e-3 if n >= 1000 else 1e-2
        np.testing.assert_allclose(res["DT_cov"][p], ref["DT_cov"][p], rtol=tol, atol=tol * np.abs(ref["DT_cov"][p]).max() + 1e-15,
                                   err_msg=f"problem {p} ({kinds[p]})")
    n_all = len(ip) + len(il)
    print(f"explicit lists: B = {B} problems on {explicit['ctas']} persistent CTAs; worst pose deviation {worst[0]:.2e} rad / "
          f"{worst[1]:.2e} m; {n_flips} of {n_all} inlier flags differ")
    assert n_flips <= max(2, n_all // 1000)
    res2, ip2, il2 = engine.optimize_pose(cam, cfg, mb)
    assert res.tobytes() + ip.tobytes() + il.tobytes() == res2.tobytes() + ip2.tobytes() + il2.tobytes()

    # the streamed form pinned: every problem's bytes equal those of the same problem solved in a batch of 5
    groups = [list(range(i, min(i + 5, B))) for i in range(0, B, 5)]
    outs, _ = _run_isolated(tmp_path, "explicit_streamed", dict(PLSTVO_STREAM_SOLVE="1"),
                            [("optimize", cam, cfg, mb)] + [("optimize", cam, cfg, _sub_matched(mb, g)) for g in groups])
    big = outs[0]
    assert big["results"].tobytes() == res.tobytes()      # the default policy chose the streamed form for this batch too
    np.testing.assert_array_equal(big["inlier_pt"], ip)
    np.testing.assert_array_equal(big["inlier_ls"], il)
    for g, out in zip(groups, outs[1:]):
        sub = _sub_matched(mb, g)
        for j, p in enumerate(g):
            a, b, c, d = mb.pt_off[p], mb.pt_off[p + 1], mb.ls_off[p], mb.ls_off[p + 1]
            e, f, h, k = sub.pt_off[j], sub.pt_off[j + 1], sub.ls_off[j], sub.ls_off[j + 1]
            assert out["results"][j].tobytes() == big["results"][p].tobytes(), (p, kinds[p])
            assert out["inlier_pt"][e:f].tobytes() == big["inlier_pt"][a:b].tobytes(), (p, kinds[p])
            assert out["inlier_ls"][h:k].tobytes() == big["inlier_ls"][c:d].tobytes(), (p, kinds[p])


# ---- 4. robust mode beyond shared memory, and at B > sm_count ----
def test_robust_mode_c5_lists_take_k2_global_scratch(engine, oracle):
    cfg = T.kitti_config()
    cfg.solver_mode = 1
    prev, curr, _, cam = synth.make_batch("hd", 3)
    gpu, ref = engine.track_batch(cam, cfg, prev, curr), oracle.track_batch(cam, cfg, prev, curr, threads=_threads())
    worst = compare(gpu, ref, prev, tight=False, flags_exact=False)
    n_diff = int((gpu["inlier_pt"] != ref["inlier_pt"]).sum() + (gpu["inlier_ls"] != ref["inlier_ls"]).sum())
    n = prev.n_pt + prev.n_ls
    print(f"robust mode, C5 lists (streamed prepare, K2 global scratch): worst pose deviation {worst}, {n_diff} of {n} flags differ")
    assert n_diff <= max(2, n // 2000)


def test_robust_mode_past_one_wave(engine, oracle, sm_count):
    cfg = T.euroc_config()
    cfg.solver_mode = 1
    B = sm_count + 20
    prev, curr, _, cam = synth.make_batch("euroc", B, first_pair=300)
    bounds = chunk_schedule(B, sm_count, False)
    assert len(bounds) > 3
    gpu, ref = engine.track_batch(cam, cfg, prev, curr), oracle.track_batch(cam, cfg, prev, curr, threads=_threads())
    worst = compare(gpu, ref, prev, tight=False, flags_exact=False)
    n_diff = int((gpu["inlier_pt"] != ref["inlier_pt"]).sum() + (gpu["inlier_ls"] != ref["inlier_ls"]).sum())
    n = prev.n_pt + prev.n_ls
    print(f"robust mode, B = {B} EuRoC pairs (K2, chunks {bounds}): worst pose deviation {worst}, {n_diff} of {n} flags differ")
    assert n_diff <= max(2, n // 2000)
    edges = {q for b in bounds[1:-1] for q in (b - 1, b)}
    groups = _groups(B, edges)
    subs = [engine.track_batch(cam, cfg, prev.select(g), curr.select(g)) for g in groups]
    _check_sub_batches(gpu, subs, groups, prev, "robust mode")


# ---- 5. one context reused across plans ----
def test_workspace_reuse_equals_fresh_context(sm_count):
    from stvo_pl_b200.engine import Engine

    def fresh(fn):
        e = Engine(0)
        try:
            return fn(e)
        finally:
            e.close()

    cfg = T.kitti_config()
    BA = 300
    assert BA > sm_count
    A = synth.make_batch("kitti", BA, first_pair=2000, n_pt=600, n_ls=150, overlap=0.9)
    small = synth.make_batch("kitti", 7, first_pair=2600, n_pt=800, n_ls=200)
    X, _, camx = synth.make_matched_batch("kitti", 40, first_pair=9)
    cfg2 = T.kitti_config()
    cfg2.min_ratio_12_p, cfg2.has_lines = 0.8, 0
    track = lambda e, b, c=cfg: e.track_batch(b[3], c, b[0], b[1])
    e = Engine(0)
    try:
        seq = [("track A", lambda x: track(x, A)),
               ("optimize_pose X", lambda x: dict(zip(("results", "inlier_pt", "inlier_ls"), x.optimize_pose(camx, cfg, X)))),
               ("track A again", lambda x: track(x, A)),
               ("track A, other ratio, no lines", lambda x: track(x, A, cfg2))]
        for label, fn in seq:
            _same_bytes(fn(e), fresh(fn), label)
        # async batches of two sizes alternating over the two workspace slots: each slot re-plans at every call
        order = [A, small, small, A, A, small]
        pinned = [(e.pinned.pin_frames(b[0]), e.pinned.pin_frames(b[1]), e.pinned_outputs(b[0]), b) for b in order]
        pending = None
        for pp, pc, out, b in pinned:
            t = e.track_batch_async(b[3], cfg, pp, pc, out)
            if pending is not None:
                e.wait(pending)
            pending = t
        e.wait(pending)
        for k, (_, _, out, b) in enumerate(pinned):
            _same_bytes(out, fresh(lambda x: track(x, b)), f"async batch {k} (B = {b[0].B})")
    finally:
        e.close()
