"""The streamed evaluator's record format held to fp64 truth on the CPU (DESIGN.md section 3, "Precision design").

The records carry every pose-independent part of a residual in fp64 before rounding (du0 = fx x/z + cx - u_obs) and the pose
as (R - I | t); the kernel adds the pose's change of the projection in fp32.  Restated with every operation rounded to fp32
(tests/stream_records.residual_delta32), that form must keep the inliers' point residual u(DT) - u_obs within 5e-6 px rms
(1e-4 px at worst: near points under large motion) of the fp64 truth on KITTI-shape problems at their true poses, and be at
least 10x more accurate (rms) than the naive fp32 form, which projects through (R | t) and subtracts the observation (two
~1000 px numbers).  Measured here: 3.2e-6 px rms against 3.5e-5 px, 11x.  Outliers (residuals of hundreds of px) are left out:
the rounding of their own du0 to fp32 dominates either form, and they do not take part in the stop tests."""
import numpy as np

import stream_records as S
from stvo_pl_b200 import synth


def _errors(B=16):
    d, nv = [], []
    mb, Ts, cam = synth.make_matched_batch("kitti", B)
    for p in range(B):
        a, b = int(mb.pt_off[p]), int(mb.pt_off[p + 1])
        P, obs, DT = mb.pt_P[a:b], mb.pt_pl_obs[a:b], Ts[p]
        truth = S.residual_truth(cam, P, obs, DT)
        inl = np.hypot(truth[:, 0], truth[:, 1]) < 5.0
        d.append(np.abs(S.residual_delta32(cam, P, obs, DT) - truth)[inl].ravel())
        nv.append(np.abs(S.residual_naive32(cam, P, obs, DT) - truth)[inl].ravel())
    return np.concatenate(d), np.concatenate(nv)


def test_delta_form_residuals_against_fp64_truth():
    d, nv = _errors()
    rms_d, rms_n = np.sqrt(np.mean(d * d)), np.sqrt(np.mean(nv * nv))
    print(f"point residual error vs fp64 over {len(d) // 2} points: delta form rms {rms_d:.2e} px, max {d.max():.2e} px; "
          f"naive fp32 rms {rms_n:.2e} px, max {nv.max():.2e} px ({rms_n / rms_d:.0f}x)")
    assert len(d) > 50000 and rms_d < 5e-6 and d.max() < 1e-4
    assert rms_n > 10 * rms_d


def test_overlap_coefficients_follow_the_reference_lambda():
    """overlap_coeffs' lambda (fp64) equals lineSegmentOverlap's in every branch, and a zero-height segment in the vertical
    branch gives +-inf, NaN only where v == sv exactly (ref_numpy.overlap restates the reference)."""
    import ref_numpy as R
    rng = np.random.default_rng(4)
    n = 2000
    spl = rng.uniform(0, 1000, (n, 2))
    kind = np.arange(n) % 5
    epl = spl + rng.uniform(-200, 200, (n, 2))
    epl[kind == 1, 0] = spl[kind == 1, 0] + rng.uniform(-0.9, 0.9, (kind == 1).sum())     # vertical
    epl[kind == 2, 1] = spl[kind == 2, 1] + rng.uniform(-0.9, 0.9, (kind == 2).sum())     # horizontal
    epl[kind == 3] = spl[kind == 3]                                                       # zero length
    epl[kind == 4, 1] = spl[kind == 4, 1]                                                 # ly == 0, |lx| < 1
    epl[kind == 4, 0] = spl[kind == 4, 0] + rng.uniform(0.1, 0.9, (kind == 4).sum())
    sp = spl + rng.normal(0, 5, (n, 2))
    sp[::7, 1] = spl[::7, 1]                                                              # v == sv exactly
    ep = epl + rng.normal(0, 5, (n, 2))
    oa, ob, oc = S.overlap_coeffs(spl, epl)
    with np.errstate(all="ignore"):
        lam = np.where(np.isinf(ob), ob * (sp[:, 1] + oc), oa * sp[:, 0] + ob * sp[:, 1] + oc)
        ov = S._overlap(lam, np.where(np.isinf(ob), ob * (ep[:, 1] + oc), oa * ep[:, 0] + ob * ep[:, 1] + oc))
        ref = R.overlap(spl, epl, sp, ep)
    zero_h = (kind == 3) | (kind == 4)
    assert np.isinf(lam[zero_h & (sp[:, 1] != spl[:, 1])]).all()
    assert np.isnan(lam[zero_h & (sp[:, 1] == spl[:, 1])]).all()
    np.testing.assert_array_equal(np.isnan(ov), np.isnan(ref))
    ok = ~np.isnan(ref)
    np.testing.assert_allclose(ov[ok], ref[ok], rtol=0, atol=1e-9)
