"""Previous-frame segments of zero height in lineSegmentOverlap's vertical branch (src/stereoFrame.cpp:515-544): zero-length
segments, and segments with |lx| < 1 and ly == 0.  There the reference's lambda = (v - sv) / ly is +-inf, NaN only where the
projected endpoint has exactly v == sv, and the overlap comes out as 0 or 1.  From the identity pose synthetic data projects
every endpoint exactly onto its previous segment's v, so every such line has a NaN lambda and every problem fails (the NaN path,
test_gpu_parity_holes.py::test_zero_length_previous_segments).  Started from a motion-model prior instead, the oracle solves
them all, which the tests assert so that they are not vacuous; K2, the streamed solver and plstvo_gn_eval_stream must follow it."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import ref_numpy as R
from stvo_pl_b200 import synth, types as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 3


def degenerate_case(orc, solver_mode=0):
    """(cam, cfg with the motion model on, MatchedBatch with zero-height previous segments, priors, #zero-length, #flat).
    The priors are the clean problems' optima moved by a small twist, so that GN takes several iterations from them."""
    cfg = T.kitti_config()
    prev, curr, _, cam = synth.make_batch("kitti", B, n_pt=200, n_ls=120, overlap=1.0)
    o = orc.track_batch(cam, cfg, prev, curr)
    m = T.matched_from_frames(prev, curr, o["m12_pt"], o["m12_ls"], cfg.lsd_scale)
    _, clean, _, _ = orc.optimize_pose(cam, cfg, m)
    rng = np.random.default_rng(13)
    spl, epl = m.ls_spl.copy(), m.ls_epl.copy()
    u = rng.random(len(spl))
    z, f = u < 0.35, (u >= 0.35) & (u < 0.6)
    epl[z] = spl[z]                                                                   # zero length
    epl[f, 1] = spl[f, 1]                                                             # ly == 0, 0 < |lx| < 1
    epl[f, 0] = spl[f, 0] + rng.uniform(0.05, 0.95, f.sum()) * rng.choice([-1.0, 1.0], f.sum())
    deg = T.MatchedBatch(pt_off=m.pt_off, ls_off=m.ls_off, pt_P=m.pt_P, pt_pl_obs=m.pt_pl_obs, pt_sigma2=m.pt_sigma2,
                         ls_sP=m.ls_sP, ls_eP=m.ls_eP, ls_le_obs=m.ls_le_obs, ls_spl=spl, ls_epl=epl, ls_sigma2=m.ls_sigma2)
    mm = T.kitti_config()
    mm.use_motion_model = 1
    mm.solver_mode = solver_mode
    pri = T.identity_priors(B)
    for p in range(B):
        tw = rng.normal(0, 1, 6) * np.array([0.02, 0.02, 0.05, 0.002, 0.002, 0.002])
        pri[p]["DT"] = clean[p]["DT_opt"].reshape(4, 4) @ synth.expmap_se3(tw)
        pri[p]["DT_cov"] = np.eye(6) * 1e-6
        pri[p]["err_norm"] = 0.2
    return cam, mm, deg, pri, int(z.sum()), int(f.sum())


def _ref_or_none():
    try:
        from oracle import ref as ref_mod
        return ref_mod.Ref() if ref_mod.available() else None
    except Exception:
        return None


def _oracle_solves_all(orc, cam, cfg, deg, pri):
    rc, res, ip, il = orc.optimize_pose(cam, cfg, deg, priors=pri)
    assert (res["good"] == 1).all(), res["good"]             # the case is not vacuous: every problem is solved
    return res, ip, il


def _same_decisions(a, b, iters=True):
    """status, verdict, inlier counts and (iters: not where b is the reference's code, which does not count) GN iterations"""
    keys = ("status", "good", "n_inliers_pt", "n_inliers_ls") + (("iters_stage1", "iters_stage2") if iters else ())
    for k in keys:
        assert int(a[k]) == int(b[k]), (k, a[k], b[k])


def test_oracle_solves_zero_height_segments_from_a_prior(oracle):
    """CPU: the oracle solves every problem from the prior in both solver modes, the lambdas at the prior are +-inf for the
    zero-height segments (overlap exactly 0 or 1, both occurring), and the reference's compiled code agrees where it is built."""
    ref = _ref_or_none()
    for mode in (0, 1):
        cam, cfg, deg, pri, nz, nf = degenerate_case(oracle, mode)
        assert nz > 100 and nf > 80
        res, ip, il = _oracle_solves_all(oracle, cam, cfg, deg, pri)
        if mode == 0:
            P = R.problem_from_matched(cam, cfg, deg, 0)
            DT = pri[0]["DT"]
            ps, pe = P.proj(P.sP @ DT[:3, :3].T + DT[:3, 3]), P.proj(P.eP @ DT[:3, :3].T + DT[:3, 3])
            with np.errstate(all="ignore"):
                ov = R.overlap(P.spl, P.epl, ps, pe)
            flat = P.spl[:, 1] == P.epl[:, 1]
            assert flat.sum() > 40 and set(np.unique(ov[flat])) == {0.0, 1.0}
        if ref is not None:
            rc, res_r, ip_r, il_r = ref.optimize_pose(cam, cfg, deg, priors=pri)
            np.testing.assert_array_equal(ip, ip_r)
            np.testing.assert_array_equal(il, il_r)
            for p in range(B):
                _same_decisions(res[p], res_r[p], iters=False)
                ang, tr = R.pose_error(res[p]["DT"], res_r[p]["DT"])
                assert ang < 1e-9 and tr < 1e-8, (mode, p, ang, tr)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["gn", "robust"])
def test_k2_follows_the_oracle_from_a_prior(engine, oracle, mode):
    """K2 (plstvo_optimize_pose, fp64 per pair) in GN and robust mode: identical flags and decisions, pose within 1e-9 rad /
    1e-8 m of the oracle and of the reference's compiled code (which reports no iteration counts)."""
    cam, cfg, deg, pri, _, _ = degenerate_case(oracle, mode)
    res_o, ip_o, il_o = _oracle_solves_all(oracle, cam, cfg, deg, pri)
    res, ip, il = engine.optimize_pose(cam, cfg, deg, priors=pri)
    ref = _ref_or_none()
    res_r = ref.optimize_pose(cam, cfg, deg, priors=pri)[1] if ref else None
    np.testing.assert_array_equal(ip, ip_o)
    np.testing.assert_array_equal(il, il_o)
    for p in range(B):
        assert np.isfinite(res[p]["DT"]).all() and res[p]["good"] == 1, res[p]
        for other in (res_o[p],) + ((res_r[p],) if res_r is not None else ()):
            ang, tr = R.pose_error(res[p]["DT"], other["DT"])
            print(f"mode {mode} pair {p}: {ang:.1e} rad, {tr:.1e} m")
            _same_decisions(res[p], other, iters=other is res_o[p])
            assert ang < 1e-9 and tr < 1e-8, (p, ang, tr)


@pytest.mark.gpu
def test_streamed_evaluator_at_the_prior(engine, oracle):
    """plstvo_gn_eval_stream at the prior poses: finite H, g, e (no NaN overlap weight) equal to the oracle's optimizeFunctions,
    and to the reference's where it is built, at fp32 level.  A zero-height segment's overlap is 0 or 1 here, so a wrong lambda
    moves H by a whole line's weight."""
    cam, cfg, deg, pri, _, _ = degenerate_case(oracle)
    DT = np.stack([pri[p]["DT"] for p in range(B)])
    H, g, e, _ = engine.gn_eval_stream(cam, cfg, deg, DT, iters=1)
    ref = _ref_or_none()
    for p in range(B):
        for other in (oracle,) + ((ref,) if ref is not None else ()):
            Ho, go, eo = other.optimize_functions(cam, cfg, deg, p, DT[p])
            assert np.isfinite(Ho).all() and np.isfinite(H[p]).all() and np.isfinite(g[p]).all() and np.isfinite(e[p])
            np.testing.assert_allclose(H[p], Ho, rtol=5e-4, atol=5e-4 * np.abs(Ho).max())
            np.testing.assert_allclose(g[p], go, rtol=5e-3, atol=5e-4 * np.abs(go).max())
            assert abs(e[p] - eo) < 5e-5 * max(1.0, abs(eo)), (p, e[p], eo)


STREAM_SCRIPT = r'''
import json, sys
import numpy as np
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/tests")
import ref_numpy as R
from stvo_pl_b200.engine import Engine
from oracle.oracle import Oracle
import test_gpu_overlap_degenerate as M
eng, orc = Engine(0), Oracle()
cam, cfg, deg, pri, _, _ = M.degenerate_case(orc)
res, ip, il = eng.optimize_pose(cam, cfg, deg, priors=pri)
rc, ro, ipo, ilo = orc.optimize_pose(cam, cfg, deg, priors=pri)
out = dict(flags=int((ip != ipo).sum() + (il != ilo).sum()), n=len(ip) + len(il), pairs=[])
for p in range(len(res)):
    ang, tr = R.pose_error(res[p]["DT"], ro[p]["DT"])
    out["pairs"].append(dict(gpu=[int(res[p][k]) for k in ("status", "good", "iters_stage1", "iters_stage2")],
                             orc=[int(ro[p][k]) for k in ("status", "good", "iters_stage1", "iters_stage2")],
                             finite=bool(np.isfinite(res[p]["DT"]).all()), ang=float(ang), tr=float(tr)))
try:
    from oracle import ref as ref_mod
    ref = ref_mod.Ref() if ref_mod.available() else None
except Exception:
    ref = None
if ref is not None:                      # the reference's compiled code: status, verdict, pose (it counts no iterations)
    rr = ref.optimize_pose(cam, cfg, deg, priors=pri)[1]
    out["ref"] = [dict(st=[int(rr[p]["status"]), int(rr[p]["good"])], gpu=[int(res[p]["status"]), int(res[p]["good"])],
                       pose=[float(x) for x in R.pose_error(res[p]["DT"], rr[p]["DT"])]) for p in range(len(res))]
print("RESULT " + json.dumps(out))
'''


@pytest.mark.gpu
def test_streamed_solver_follows_the_oracle_from_a_prior():
    """The same problems through the streamed solver (forced with PLSTVO_STREAM_SOLVE=1, read when the library loads, hence
    the subprocess): the oracle's status, verdict and iteration counts, pose within 1e-5 rad / 1e-4 m, also against the
    reference's compiled code where it is built."""
    env = dict(os.environ, PLSTVO_STREAM_SOLVE="1")
    r = subprocess.run([sys.executable, "-c", "ROOT = %r\n" % ROOT + STREAM_SCRIPT], capture_output=True, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])
    print(out)
    assert out["flags"] <= 2, out
    for rec in out["pairs"]:
        assert rec["orc"][1] == 1, rec                                   # not vacuous
        assert rec["finite"] and rec["gpu"] == rec["orc"], rec
        assert rec["ang"] < 1e-5 and rec["tr"] < 1e-4, rec
    for rec in out.get("ref", []):
        assert rec["st"] == rec["gpu"] and rec["pose"][0] < 1e-5 and rec["pose"][1] < 1e-4, rec
