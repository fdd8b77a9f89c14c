"""session_keyframe_kernel (keyframe.cu), the key-frame test every session run with the test launches, on placed inputs
through plstvo_debug_keyframe: the shipped kernel against the 60-digit needNewKF of hp_keyframe.py, the reference's own
needNewKF compiled into oracle/_ref (the reference's text on the stand-in's LU, not Eigen; where built), plstvo.hpp's
KeyframeTest and handler.KeyframeTest, on every case of hp_keyframe.cases (test_keyframe_decisions_host.py holds the host
implementations to the same assertions).

Held: the decision and counter are the exact ones wherever the exact values lie outside their bands (t at its threshold and
one ulp either side with t exactly 5 2^k; r, t and the ratio at 4 bounds either side; the counter at 10 and 11 and over 12
chained calls); the diagnostics and the returned state within hp_keyframe's bounds; new_kf follows from the kernel's own
diagnostics and counter; where the inputs are non-finite the reference library's decision, counter and NaN / inf pattern.
Launch shapes n = 1, 63, 64, 65 and 64 SMs + 5 with the cases mixed: each stream's output, state and prior equal, byte for
byte, those of a launch of its own; fired streams' priors take Tfw = I and Tfw_cov = I, every other byte is kept."""
import numpy as np
import pytest

import hp_keyframe as hk
from test_gpu_track_images import sm_count
from test_keyframe_decisions_host import CASES, Ratios, build_cpp, check, ref_lib, run_cpp, run_handler, run_ref
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


def results_of(items):
    """PlPoseResult records carrying each (Tfw, DT, DT_cov); every other byte is a sentinel the kernel must not need."""
    r = np.frombuffer(bytes([0x5A]) * (len(items) * T.POSE_RESULT_DTYPE.itemsize), T.POSE_RESULT_DTYPE).copy()
    for i, (Tfw, DT, cov) in enumerate(items):
        r["Tfw"][i], r["DT"][i], r["DT_cov"][i] = np.reshape(Tfw, (4, 4)), np.reshape(DT, (4, 4)), np.reshape(cov, (6, 6))
    return r


def sentinel_priors(n):
    return np.frombuffer(bytes([SENTINEL]) * (n * T.PRIOR_DTYPE.itemsize), T.PRIOR_DTYPE).copy()


def run_device(e, cases):
    """All cases at once, one hook call per step (the cases with a step t in one launch): per case the rows
    [(result row, entropy_first_prevKF, cov_prevKF_currF)] as the state stands after each call."""
    states = [c["state"].copy() for c in cases]
    rows = [[] for _ in cases]
    for t in range(max(len(c["steps"]) for c in cases)):
        live = [i for i, c in enumerate(cases) if t < len(c["steps"])]
        for k in sorted({cases[i]["k"] for i in live}):
            idx = [i for i in live if cases[i]["k"] == k]
            st = np.concatenate([states[i] for i in idx])
            out = e.debug_keyframe(np.array([k], T.KEYFRAME_CONFIG_DTYPE), results_of([cases[i]["steps"][t] for i in idx]), st)
            for j, i in enumerate(idx):
                states[i] = st[j:j + 1].copy()
                rows[i].append((out[j], float(st["entropy_first_prevKF"][j]), np.array(st["cov_prevKF_currF"][j])))
    return rows


@pytest.fixture(scope="module")
def engine():
    e = Engine()
    yield e
    e.close()


@pytest.fixture(scope="module")
def cpp_exe(tmp_path_factory):
    return build_cpp(str(tmp_path_factory.mktemp("kfd")))


def test_every_case_against_the_restatement_and_the_reference(engine, cpp_exe):
    lib = ref_lib()
    dev = run_device(engine, CASES)
    ratios = Ratios()
    for c, rows in zip(CASES, dev):
        ref_rows = run_ref(lib, c) if lib else None
        check("device", c, rows, ratios, ref_rows)
        # the host implementations on the same case, for the record of one run (test_keyframe_decisions_host.py holds them)
        check("plstvo.hpp", c, run_cpp(cpp_exe, c), Ratios(), ref_rows)
        check("handler.py", c, run_handler(c), Ratios(), ref_rows)
        if ref_rows is not None:   # step by step, the reference's decision and counter wherever no band decides
            want = hk.run(c["k"], c["state"], c["steps"])
            for i, ((g, _, _), (r, _, _)) in enumerate(zip(rows, ref_rows)):
                if i >= len(want) or (want[i] is not None and want[i]["fire"] is None):
                    break
                assert (int(g["new_kf"]), int(g["N_prevKF_currF"])) == (int(r["new_kf"]), int(r["N_prevKF_currF"])), \
                    (c["label"], i, g, r)
    print("device error / bound:", ratios)


def test_counter_over_chained_calls(engine):
    """11 quiet steps and a 12th that fires, one hook call each, from the initial state."""
    c = next(c for c in CASES if c["label"] == "counter chain")
    rows = run_device(engine, [c])[0]
    assert [int(r["new_kf"]) for r, _, _ in rows] == [0] * 11 + [1]
    assert [int(r["N_prevKF_currF"]) for r, _, _ in rows] == list(range(1, 12)) + [11]


@pytest.mark.parametrize("n", [1, 63, 64, 65, "sms"])
def test_launch_shapes(engine, n):
    n = 64 * sm_count() + 5 if n == "sms" else n
    pick = [CASES[(7 * j) % len(CASES)] for j in range(n)]
    k = np.array([(0.85, 5.0, 15.0)], T.KEYFRAME_CONFIG_DTYPE)
    st = np.concatenate([c["state"] for c in pick])
    pri = sentinel_priors(n)
    out = engine.debug_keyframe(k, results_of([c["steps"][0] for c in pick]), st, pri)
    solo = {}
    for c in {id(c): c for c in pick}.values():
        s1, p1 = c["state"].copy(), sentinel_priors(1)
        o1 = engine.debug_keyframe(k, results_of([c["steps"][0]]), s1, p1)
        solo[id(c)] = (o1.tobytes(), s1.tobytes(), p1.tobytes())
    fresh = sentinel_priors(1)
    for j, c in enumerate(pick):
        assert (out[j:j + 1].tobytes(), st[j:j + 1].tobytes(), pri[j:j + 1].tobytes()) == solo[id(c)], (n, j, c["label"])
        if out["new_kf"][j]:
            assert np.array_equal(pri["Tfw"][j], np.eye(4)) and np.array_equal(pri["Tfw_cov"][j], np.eye(6))
            for f in ("DT", "DT_cov", "err_norm"):
                assert pri[j:j + 1][f].tobytes() == fresh[f].tobytes(), (j, f)
        else:
            assert pri[j:j + 1].tobytes() == fresh.tobytes(), j
    if n > 1:
        assert out["new_kf"].any() and not out["new_kf"].all()


def test_priors_may_be_null_and_n_zero(engine):
    c = CASES[0]
    s = c["state"].copy()
    out = engine.debug_keyframe(np.array([c["k"]], T.KEYFRAME_CONFIG_DTYPE), results_of([c["steps"][0]]), s)
    s2, p2 = c["state"].copy(), sentinel_priors(1)
    out2 = engine.debug_keyframe(np.array([c["k"]], T.KEYFRAME_CONFIG_DTYPE), results_of([c["steps"][0]]), s2, p2)
    assert out.tobytes() == out2.tobytes() and s.tobytes() == s2.tobytes()
    assert len(engine.debug_keyframe(np.array([c["k"]], T.KEYFRAME_CONFIG_DTYPE), results_of([]),
                                     np.zeros(0, T.KEYFRAME_STATE_DTYPE))) == 0
