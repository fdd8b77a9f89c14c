"""The key-frame test's fp64 implementations on the host, held to the 60-digit needNewKF of hp_keyframe.py on placed cases
(hp_keyframe.cases: t, r and the entropy ratio at their thresholds, the counter, first steps, degenerate covariances and
non-finite poses): the reference's own needNewKF / currFrameIsKF compiled into oracle/_ref (the reference's text on the
stand-in's LU, not Eigen; skipped where the library is absent), plstvo.hpp's KeyframeTest and handler.KeyframeTest.

Each implementation's diagnostics and state (cov_prevKF_currF, entropy_first_prevKF) lie within hp_keyframe's bounds, its
counter is exact, and its decision is the exact one wherever the exact values lie outside their bands.  Where the inputs are
non-finite (an fp64 artefact the 60-digit restatement does not model) the reference library's fp64 result is the answer:
decisions, counters and the NaN / inf pattern of every diagnostic equal it.  Every decision also follows from the
implementation's own diagnostics and counter."""
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import hp_keyframe as hk
from stvo_pl_b200 import types as T
from stvo_pl_b200.handler import HandlerConfig, KeyframeTest

FIELDS = ("e_curr", "ratio", "t", "r")
ROW = {"e_curr": "entropy_curr", "ratio": "entropy_ratio", "t": "t", "r": "r"}

CPP_HELPER = r'''#include <cstdio>
#include "plstvo.hpp"
// stdin: PlKeyframeConfig, PlKeyframeState, int32 T, then T records of Tfw [16], DT [16], DT_cov [36].  Prints, per step, the
// decision, N_prevKF_currF, entropy_curr, entropy_ratio, t, r, then the state after currFrameIsKF: entropy_first_prevKF and
// cov_prevKF_currF [36] (%a: exact)
int main() {
    PlKeyframeConfig k;
    PlKeyframeState s;
    int32_t T;
    if (std::fread(&k, sizeof k, 1, stdin) != 1 || std::fread(&s, sizeof s, 1, stdin) != 1 || std::fread(&T, 4, 1, stdin) != 1)
        return 2;
    plstvo::HandlerConfig hc;
    hc.min_entropy_ratio = k.min_entropy_ratio; hc.max_kf_t_dist = k.max_kf_t_dist; hc.max_kf_r_dist = k.max_kf_r_dist;
    plstvo::KeyframeTest kt = plstvo::KeyframeTest::fromState(s);
    for (int t = 0; t < T; ++t) {
        double rec[68];
        if (std::fread(rec, sizeof rec, 1, stdin) != 1) return 2;
        plstvo::StereoFrame f;
        std::copy(rec, rec + 16, f.Tfw.begin());
        std::copy(rec + 16, rec + 32, f.DT.begin());
        std::copy(rec + 32, rec + 68, f.DT_cov.begin());
        const bool kf = kt.needNewKF(hc, f);
        std::printf("%d %d %a %a %a %a", kf ? 1 : 0, kt.N_prevKF_currF, kt.entropy_curr, kt.entropy_ratio, kt.kf_t, kt.kf_r);
        if (kf) kt.currFrameIsKF(f);
        std::printf(" %a", kt.entropy_first_prevKF);
        for (double v : kt.cov_prevKF_currF) std::printf(" %a", v);
        std::printf("\n");
    }
    return 0;
}
'''


def build_cpp(d) -> str:
    src = os.path.join(d, "kfd.cpp")
    with open(src, "w") as f:
        f.write(CPP_HELPER)
    exe = os.path.join(d, "kfd")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"),
                    src, "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def cpp_exe(tmp_path_factory):
    return build_cpp(str(tmp_path_factory.mktemp("kfd")))


def _row(fire, N, e, q, t, r):
    o = np.zeros(1, T.KEYFRAME_RESULT_DTYPE)[0]
    o["new_kf"], o["N_prevKF_currF"], o["entropy_curr"], o["entropy_ratio"], o["t"], o["r"] = int(fire), N, e, q, t, r
    return o


def run_cpp(exe, case):
    """plstvo.hpp's KeyframeTest over the case: [(result row, entropy_first_prevKF, cov_prevKF_currF)] per step."""
    k = np.array([case["k"]], T.KEYFRAME_CONFIG_DTYPE)
    blob = k.tobytes() + case["state"].tobytes() + np.int32(len(case["steps"])).tobytes()
    for Tfw, DT, cov in case["steps"]:
        blob += np.concatenate([np.ravel(Tfw), np.ravel(DT), np.ravel(cov)]).astype(np.float64).tobytes()
    out = subprocess.run([exe], input=blob, capture_output=True, check=True).stdout.decode().splitlines()
    rows = []
    for ln in out:
        v = ln.split()
        f = [float.fromhex(x) for x in v[2:]]
        rows.append((_row(int(v[0]), int(v[1]), *f[:4]), f[4], np.array(f[5:]).reshape(6, 6)))
    return rows


def run_handler(case):
    kt = KeyframeTest.from_state(case["state"])
    c = HandlerConfig(min_entropy_ratio=case["k"][0], max_kf_t_dist=case["k"][1], max_kf_r_dist=case["k"][2])
    rows = []
    for Tfw, DT, cov in case["steps"]:
        fire = kt.needNewKF(c, Tfw, DT, cov)
        row = _row(fire, kt.N_prevKF_currF, kt.entropy_curr, kt.entropy_ratio, kt.t, kt.r)
        if fire:
            kt.currFrameIsKF(type("F", (), {})())
        rows.append((row, float(kt.entropy_first_prevKF), np.array(kt.cov_prevKF_currF, float)))
    return rows


def ref_lib():
    """The reference library, or None where it is absent or was built (elsewhere) by a recipe without the key-frame entry."""
    from oracle import ref
    if not ref.available():
        return None
    lib = ref.Ref()
    return lib if lib.has_need_new_kf else None


def run_ref(lib, case):
    s = case["state"].copy()
    rows = []
    for Tfw, DT, cov in case["steps"]:
        row = lib.need_new_kf(np.array([case["k"]], T.KEYFRAME_CONFIG_DTYPE), s, Tfw, DT, cov)[0]
        rows.append((row, float(s["entropy_first_prevKF"][0]), np.array(s["cov_prevKF_currF"][0])))
    return rows


def pattern(v) -> str:
    return "nan" if math.isnan(v) else ("+inf" if v == math.inf else ("-inf" if v == -math.inf else "finite"))


class Ratios:
    """The largest error-to-bound ratio seen per quantity."""
    def __init__(self):
        self.m = {}

    def add(self, name, err, bound):
        if bound > 0:
            self.m[name] = max(self.m.get(name, 0.0), err / bound)

    def __str__(self):
        return ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.m.items()))


def follows(case, i, row):
    """new_kf from the implementation's own diagnostics and counter (the counter before needNewKF's increment)."""
    mr, mt, mx = case["k"]
    q = float(row["entropy_ratio"])
    DT, cov = np.asarray(case["steps"][i][1]), np.asarray(case["steps"][i][2])
    n_before = int(row["N_prevKF_currF"]) - (0 if row["new_kf"] else 1)
    want = (q < mr or math.isnan(q) or math.isinf(q) or (not cov.any() and np.array_equal(DT.reshape(4, 4), np.eye(4)))
            or float(row["t"]) > mt or float(row["r"]) > mx or n_before > 10)
    return int(want) == int(row["new_kf"])


def check(name, case, rows, ratios, ref_rows=None):
    """One implementation's rows [(row, entropy_first, cov)] against the restatement, and against the reference library's
    rows where the restatement stops at an fp64 artefact."""
    want = hk.run(case["k"], case["state"], case["steps"])
    for i, (row, ef, cov) in enumerate(rows):
        what = (name, case["label"], i)
        assert follows(case, i, row), what + (row,)
        if i >= len(want):
            break
        o = want[i]
        if o is None:
            if ref_rows is not None:
                r = ref_rows[i][0]
                assert (int(row["new_kf"]), int(row["N_prevKF_currF"])) == (int(r["new_kf"]), int(r["N_prevKF_currF"])), \
                    what + (row, r)
                for f in ("entropy_ratio", "t", "r") + (() if r["new_kf"] else ("entropy_curr",)):
                    assert pattern(float(row[f])) == pattern(float(r[f])), what + (f, row, r)
                    if pattern(float(r[f])) == "finite":
                        assert float(row[f]) == pytest.approx(float(r[f]), rel=1e-9, abs=1e-12), what + (f, row, r)
                assert pattern(ef) == pattern(ref_rows[i][1]), what + (ef, ref_rows[i][1])
            break
        for f in FIELDS:
            if f == "e_curr" and name == "reference" and row["new_kf"]:
                continue                                 # the reference's firing line does not print it
            got, ex, b = float(row[ROW[f]]), o[f], o["b_" + ("e" if f == "e_curr" else f)]
            if math.isfinite(ex):
                err = abs(got - ex)
                assert err <= b, what + (f, got, ex, b)
                ratios.add(f, err, b)
            else:
                assert pattern(got) == pattern(ex), what + (f, got, ex)
        if math.isfinite(o["e_first"]):                  # currFrameIsKF leaves entropy_first_prevKF as needNewKF set it
            assert abs(ef - o["e_first"]) <= o["b_first"], what + ("e_first", ef, o["e_first"], o["b_first"])
            ratios.add("e_first", abs(ef - o["e_first"]), o["b_first"])
        else:
            assert pattern(ef) == pattern(o["e_first"]), what + ("e_first", ef, o["e_first"])
        if not o["fire"]:
            err = np.abs(cov - o["cov"])
            assert (err <= o["b_cov"]).all(), what + ("cov", float((err - o["b_cov"]).max()))
            nz = o["b_cov"] > 0
            if nz.any():
                ratios.add("cov", float((err[nz] / o["b_cov"][nz]).max()), 1.0)
        elif o["fire"]:
            assert not cov.any(), what + ("cov after currFrameIsKF",)
        if o["fire"] is None:
            break
        assert int(row["new_kf"]) == int(o["fire"]) and int(row["N_prevKF_currF"]) == o["N"], what + (row, o["fire"], o["N"])


CASES = hk.cases()


def test_cases_cover_every_branch():
    """The placed cases decide every criterion both ways, and leave the band cases to no one."""
    fired = [hk.run(c["k"], c["state"], c["steps"]) for c in CASES]
    decided = [o["fire"] for r in fired for o in r if o is not None]
    assert True in decided and False in decided and None not in decided
    assert sum(o is None for r in fired for o in r) >= 12   # the artefact cases, decided by the reference library


def test_reference_library_against_the_restatement():
    lib = ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref not built with the key-frame entry (the reference checkout is absent)")
    ratios = Ratios()
    for c in CASES:
        check("reference", c, run_ref(lib, c), ratios)
    print("reference:", ratios)


def test_plstvo_hpp_against_the_restatement_and_the_reference(cpp_exe):
    lib = ref_lib()
    ratios = Ratios()
    for c in CASES:
        check("plstvo.hpp", c, run_cpp(cpp_exe, c), ratios, run_ref(lib, c) if lib else None)
    print("plstvo.hpp:", ratios)


def test_handler_against_the_restatement_and_the_reference():
    lib = ref_lib()
    ratios = Ratios()
    for c in CASES:
        check("handler.py", c, run_handler(c), ratios, run_ref(lib, c) if lib else None)
    print("handler.py:", ratios)


def test_the_two_confirmed_differences_follow_the_reference(cpp_exe):
    """A NaN cosine in logmap stays NaN (r = 0, so a negative max_kf_r_dist fires), and a zero pivot with inf below it gives a
    NaN determinant (entropy_first_prevKF NaN, not -999999999.99): pinned on both mirrors, and on the reference where built."""
    nan_r = next(c for c in CASES if c["label"] == "Tfw NaN R max_r -1")
    piv = next(c for c in CASES if c["label"] == "first zero pivot then inf")
    impls = [run_handler, lambda c: run_cpp(cpp_exe, c)]
    lib = ref_lib()
    if lib is not None:
        impls.append(lambda c: run_ref(lib, c))
    for run in impls:
        row = run(nan_r)[0][0]
        assert row["new_kf"] == 1 and row["r"] == 0.0 and math.isnan(row["t"]), row
        assert math.isnan(run(piv)[0][1])   # entropy_first_prevKF after the step (it fired, so currFrameIsKF left it)
