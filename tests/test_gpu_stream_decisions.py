"""The streamed GN loop's decisions at its thresholds (gn_loop_stream_kernel, solve.cu): close calls and hand-offs.

One problem per call (B = 1), forced onto the streamed solver (PLSTVO_STREAM_SOLVE=1 is read when the library loads, hence the
subprocess).  Thresholds are placed per case from an fp64 trace of the oracle's Gauss-Newton iterations (ref_numpy.Problem,
instrumented below), and the oracle's own iteration counts confirm that the two signs of each offset stop at different
iterations:

* min_error close calls: min_error = err_k (1 +- d) for a stage-2 iteration k, above every stage-1 error;
* min_error_change close calls: min_error_change = (err_{k-1} - err_k) +- d err_k, where neither the increment test nor an
  earlier error test fires first;
* increment hand-offs: min_error_change = max(|inc_t|, |inc_r|) of stage 1's first increment times (1 +- d_inc), d_inc inside
  GL_INC_BAND (1e-3): the streamed solver hands the problem to K2, the fp64 kernel.  Only there can the increment test decide
  (later, the error changes are far below the increments and the error test fires first), and that increment comes from the
  first evaluation at the start pose, so its noise is the fp32 evaluation's (~1e-6 relative, test_gpu_stream_precision.py),
  far inside d_inc = GL_INC_BAND / 3.

Before placing d, each candidate's noise floor is measured: the GPU runs the problem with max_iters_ref = k (and k - 1), and
the fp64 error at its DT_opt (oracle.optimize_functions, stage-2 inlier flags) is compared, relative to err_k, with the same at
the oracle's.  Each case sits at the first iteration whose floor is at most a sixth of GL_ERR_BAND (2e-6 err), and d sweeps
band / 4 and band / 2 where they are at least 3x the floor (the other half of the band holds the fp32-summed error's own
deviation from fp64, measured up to ~4e-7 of err).  Asserted: the oracle's status, verdict and both
iteration counts for both signs; for d inside the band, a non-zero close-call slot of plstvo_batch_phase_cycles (the fp64
path ran); for hand-offs, delegated_to_fp64 > 0 and result bytes equal to the same input under PLSTVO_STREAM_SOLVE=0."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import ref_numpy as R
from stvo_pl_b200 import synth, types as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GL_ERR_BAND, GL_INC_BAND = 2e-6, 1e-3
CLOSE_SLOT = [8 + 11 * s + 5 for s in (0, 1)]          # GLP_FIRST + GLP_N s + GLP_CLOSE (include/plstvo.h)
FIRST_PAIRS = (0, 1, 2)


class Traced(R.Problem):
    """ref_numpy.Problem whose GN calls record (err, err_prev, |inc_t|, |inc_r|) per iteration, one list per call."""

    def __init__(self, *a):
        super().__init__(*a)
        self.trace = []

    def gn(self, DT, max_iters):
        cfg, rec = self.cfg, []
        self.trace.append(rec)
        err_prev = 999999999.9
        self.evals = 0
        H = np.zeros((6, 6))
        err = 0.0
        for it in range(max_iters):
            H, g, err = self.evaluate(DT)
            rec.append(dict(err=err, err_prev=err_prev))
            if err > err_prev:
                if it > 0:
                    break
                return DT, None, -1.0
            if err < cfg.min_error or abs(err - err_prev) < cfg.min_error_change:
                break
            inc = np.linalg.solve(H, g)
            rec[-1].update(nt=float(np.linalg.norm(inc[:3])), nr=float(np.linalg.norm(inc[3:])))
            DT = DT @ R.inverse_se3(R.expmap_se3(inc))
            if np.linalg.norm(inc[:3]) < cfg.min_error_change and np.linalg.norm(inc[3:]) < cfg.min_error_change:
                break
            err_prev = err
        return DT, np.linalg.inv(H), err


def problem(orc, first_pair):
    """(cam, cfg, prev, curr, matched) of one KITTI-shape pair"""
    cfg = T.kitti_config()
    prev, curr, _, cam = synth.make_batch("kitti", 1, first_pair=first_pair, n_pt=600, n_ls=150)
    o = orc.track_batch(cam, cfg, prev, curr)
    m = T.matched_from_frames(prev, curr, o["m12_pt"], o["m12_ls"], cfg.lsd_scale)
    return cam, cfg, prev, curr, m


def trace(cam, cfg, m):
    P = Traced(cam, cfg, m.pt_P, m.pt_pl_obs, m.pt_sigma2, m.ls_sP, m.ls_eP, m.ls_le_obs, m.ls_spl, m.ls_epl, m.ls_sigma2)
    out = P.optimize_pose()
    return P.trace, out


def with_cfg(cfg, **kw):
    c = T.PlConfig()
    C_fields = [f[0] for f in T.PlConfig._fields_]
    for f in C_fields:
        setattr(c, f, getattr(cfg, f))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _iters(res):
    return [int(res[k][0]) for k in ("status", "good", "iters_stage1", "iters_stage2")]


def candidates(orc, cam, cfg, prev, curr, m):
    """The cases of one problem: [(kind, k, field, base, scale)], threshold = base + sign * d * scale, each confirmed on the
    oracle to stop at different iterations for the two signs (at d = GL_ERR_BAND / 2, or GL_INC_BAND / 3 for hand-offs),
    with stage 1 as without the offset."""
    tr, out = trace(cam, cfg, m)
    if out["status"] != 0 or len(tr) != 2:
        return []
    s1, s2 = tr
    base_it1 = _iters(orc.track_batch(cam, cfg, prev, curr)["results"])[2]
    s1_min = min(r["err"] for r in s1)
    cases = []
    for k in range(1, len(s2)):
        ek = s2[k]["err"]
        if ek < s1_min * (1 - 1e-4):
            cases.append(("min_error", k, "min_error", ek, ek))
        d = s2[k]["err_prev"] - ek
        inc_prev = max(s2[k - 1].get("nt", 0.0), s2[k - 1].get("nr", 0.0))
        earlier = min(abs(s2[j]["err_prev"] - s2[j]["err"]) for j in range(1, k + 1))
        if d > 0 and inc_prev > 2 * d and earlier >= d:
            cases.append(("min_error_change", k, "min_error_change", d, ek))
    # the increment test decides only where the error test cannot fire first: at stage 1's first iteration (err_prev is the
    # reference's 999999999.9); its increment does not depend on any threshold
    big, small = max(s1[0]["nt"], s1[0]["nr"]), min(s1[0]["nt"], s1[0]["nr"])
    if small < big * (1 - 3 * GL_INC_BAND):
        cases.append(("handoff", 0, "min_error_change", big, big))
    good = []
    for kind, k, field, base, scale in cases:
        d = GL_INC_BAND / 3 if kind == "handoff" else GL_ERR_BAND / 2
        r = [_iters(orc.track_batch(cam, with_cfg(cfg, **{field: base + s * d * scale}), prev, curr)["results"]) for s in (1, -1)]
        if kind == "handoff":
            ok = r[0][2] != r[1][2]                                # stage 1 stops after its first or its second iteration
        else:
            ok = r[0][2] == r[1][2] == base_it1 and r[0][3] != r[1][3] and r[0][0] == r[1][0] == 0
        if ok:
            good.append((kind, k, field, base, scale))
    return good


SCRIPT = r'''
import json, sys
import numpy as np
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/tests")
from stvo_pl_b200.engine import Engine
from stvo_pl_b200 import types as T
from oracle.oracle import Oracle
import test_gpu_stream_decisions as M
eng, orc = Engine(0), Oracle()
jobs = json.loads(sys.argv[1])
out = []
def run(cam, cfg, prev, curr, phases):
    db = eng.upload(cam, cfg, prev, curr)
    try:
        db.run()
        res = db.download()
        st = db.stage_times(1)
        cyc = db.phase_cycles()[0].tolist() if phases else None
    finally:
        db.free()
    return res, st, cyc
for job in jobs:
    cam, cfg, prev, curr, m = M.problem(orc, job["pair"])
    rec = dict(job)
    if job["what"] == "floor":
        fl = []
        for k in job["ks"]:
            c = M.with_cfg(cfg, max_iters_ref=k)
            g, _, _ = run(cam, c, prev, curr, False)
            r = orc.track_batch(cam, c, prev, curr)
            mm = M.stage2_lists(m, r)
            eg = orc.optimize_functions(cam, cfg, mm, 0, g["results"]["DT_opt"][0])[2]
            eo = orc.optimize_functions(cam, cfg, mm, 0, r["results"]["DT_opt"][0])[2]
            fl.append(abs(eg - eo) / abs(eo))
        rec["floor"] = max(fl)
    else:
        c = M.with_cfg(cfg, **{job["field"]: job["value"]})
        g, st, cyc = run(cam, c, prev, curr, True)
        r = orc.track_batch(cam, c, prev, curr)
        rec.update(gpu=M._iters(g["results"]), orc=M._iters(r["results"]), delegated=st["delegated_to_fp64"],
                   streamed=st["streamed_solver"], close=[cyc[s] for s in M.CLOSE_SLOT], bytes=g["results"].tobytes().hex())
    out.append(rec)
print("RESULT " + json.dumps(out))
'''


def stage2_lists(m, r):
    """the matched lists with the stage-2 inlier flags of a track result (the flags of the matched features, in order)"""
    ip = r["inlier_pt"][r["m12_pt"] >= 0]
    il = r["inlier_ls"][r["m12_ls"] >= 0]
    return T.MatchedBatch(pt_off=m.pt_off, ls_off=m.ls_off, pt_P=m.pt_P, pt_pl_obs=m.pt_pl_obs, pt_sigma2=m.pt_sigma2,
                          ls_sP=m.ls_sP, ls_eP=m.ls_eP, ls_le_obs=m.ls_le_obs, ls_spl=m.ls_spl, ls_epl=m.ls_epl,
                          ls_sigma2=m.ls_sigma2, pt_inlier=ip, ls_inlier=il)


def _run(jobs, stream):
    env = dict(os.environ, PLSTVO_STREAM_SOLVE="1" if stream else "0")
    r = subprocess.run([sys.executable, "-c", "ROOT = %r\n" % ROOT + SCRIPT, json.dumps(jobs)], capture_output=True, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])


@pytest.mark.gpu
def test_close_calls_and_handoffs_follow_the_oracle(oracle):
    cases = []
    for fp in FIRST_PAIRS:
        cam, cfg, prev, curr, m = problem(oracle, fp)
        cases += [(fp,) + c for c in candidates(oracle, cam, cfg, prev, curr, m)]
    assert {c[1] for c in cases} == {"min_error", "min_error_change", "handoff"}, cases
    # every error-test candidate's noise floor; per problem and kind, the first iteration whose floor the band holds (early
    # iterations take large steps: their error is first-order in the trajectory's difference, and their floor is larger)
    need = [c for c in cases if c[1] != "handoff"]
    floors = _run([dict(what="floor", pair=fp, kind=kind, k=k, ks=[k - 1, k] if k > 1 else [k]) for fp, kind, k, *_ in need], True)
    floor_of = {(f["pair"], f["kind"], f["k"]): f["floor"] for f in floors}
    for f in floors:
        print(f"floor {f['kind']} pair {f['pair']} k {f['k']}: {f['floor']:.1e}")
    chosen, seen = [], set()
    for c in cases:
        fp, kind, k = c[:3]
        if (fp, kind) not in seen and (kind == "handoff" or 3 * floor_of[(fp, kind, k)] <= GL_ERR_BAND / 2):
            seen.add((fp, kind))
            chosen.append(c)
    assert {c[1] for c in chosen} == {"min_error", "min_error_change", "handoff"}, (chosen, floors)
    jobs = []
    for fp, kind, k, field, base, scale in chosen:
        floor = floor_of.get((fp, kind, k), 0.0)
        if kind == "handoff":
            ds = [GL_INC_BAND / 3]
        else:
            # the half band beyond the offset holds the fp32-summed error's own deviation (up to ~4e-7 of err measured)
            ds = [d for d in (GL_ERR_BAND / 4, GL_ERR_BAND / 2) if d >= 3 * floor]
        for d in ds:
            for s in (1, -1):
                jobs.append(dict(what="case", pair=fp, kind=kind, k=k, field=field, value=base + s * d * scale, d=d, sign=s,
                                 floor=floor))
    res = _run(jobs, True)
    handoffs = [j for j in res if j["kind"] == "handoff"]
    k2_jobs = [{k: j[k] for k in ("what", "pair", "kind", "k", "field", "value")} for j in handoffs]
    k2 = {json.dumps([j["pair"], j["value"]]): j for j in _run(k2_jobs, False)}
    n_close = 0
    for j in res:
        print({k: v for k, v in j.items() if k != "bytes"})
        assert j["streamed"] and j["gpu"] == j["orc"], j                     # status, good, iters_stage1, iters_stage2
        if j["kind"] == "handoff":
            assert j["delegated"] > 0, j
            assert j["bytes"] == k2[json.dumps([j["pair"], j["value"]])]["bytes"], j
        else:
            assert j["close"][1] > 0, j                                     # stage 2 took the fp64 re-decision
            n_close += 1
    # the two signs of each offset stop at different iterations (checked on the oracle when the cases were chosen)
    for a, b in zip(res[0::2], res[1::2]):
        assert a["orc"][2:] != b["orc"][2:], (a, b)
    print(f"{len(res)} threshold runs, {n_close} close calls, {len(handoffs)} hand-offs, delegated counts "
          f"{[j['delegated'] for j in handoffs]}; cases (pair, kind, k) {[c[:3] for c in chosen]}")
