"""The streamed solver's cycle counters (plstvo_batch_phase_cycles): the timed instantiation of the GN loop
kernel computes exactly what the shipped one computes on bench.py's C2 workload, and every phase it times is counted."""
import os

import numpy as np
import pytest

from bench import make_workload, workload_config

GL_FIRST, GL_N = 8, 11
# wait, eval, fold, barrier, tests, solve, increment, trailing, inv6 (the close-call slot only counts where a close call happened)
ALWAYS = [0, 1, 2, 3, 4, 6, 7, 8, 9]


def _same(a, b):
    for k in ("m12_pt", "m12_ls", "inlier_pt", "inlier_ls"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    assert a["results"].tobytes() == b["results"].tobytes()


@pytest.mark.gpu
def test_phase_pass_matches_plain_pass(engine):
    prev, curr, _, cam = make_workload(512, 0)
    db = engine.upload(cam, workload_config(), prev, curr)
    try:
        db.run()
        plain = db.download()
        cyc = db.phase_cycles()
        timed = db.download()
        _same(plain, timed)
        db.kernel_times(iters=1)           # a pass after the timed one computes the same again
        _same(plain, db.download())
    finally:
        db.free()
    res = plain["results"]
    streamed = (cyc[:, :GL_FIRST] == 0).all(axis=1)     # the fused kernel's slots count only the problems handed back to it
    assert streamed.sum() > 400
    iters = cyc[:, [GL_FIRST + GL_N - 1, GL_FIRST + 2 * GL_N - 1]]
    np.testing.assert_array_equal(iters[streamed, 0], res["iters_stage1"][streamed])
    np.testing.assert_array_equal(iters[streamed, 1], res["iters_stage2"][streamed])
    solved = np.flatnonzero(streamed & (res["good"] == 1) & (res["iters_stage2"] > 0))
    assert len(solved) > 400
    for s in range(2):
        blk = cyc[solved, GL_FIRST + s * GL_N: GL_FIRST + (s + 1) * GL_N]
        assert (blk[:, ALWAYS] > 0).all(), (s, blk[:, ALWAYS].min(axis=0))
