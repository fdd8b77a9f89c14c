"""tools/probe_solver_phases.py without a device: its arguments parse, it makes its output directory, and its tables and trace
report come out right on made-up counters and kernel lists."""
import os
import subprocess
import sys

import numpy as np

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import probe_solver_phases as P  # noqa: E402


def test_help_parses():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "probe_solver_phases.py"), "--help"],
                       capture_output=True, text=True)
    assert r.returncode == 0 and "--out" in r.stdout and "--mode" in r.stdout
    a = P.parse_args(["--mode", "trace", "--pairs", "8"])
    assert a.mode == "trace" and a.pairs == 8 and a.out is None


def test_output_dir(tmp_path):
    d = P.output_dir(str(tmp_path / "a" / "b"))
    assert os.path.isdir(d) and d == str(tmp_path / "a" / "b")
    assert P.output_dir(d) == d                       # an existing directory is reused
    t = P.output_dir(None)
    assert os.path.isdir(t)
    os.rmdir(t)


def test_phase_table():
    cyc = np.zeros((3, 32), np.int64)
    cyc[:2, P.GL_FIRST: P.GL_FIRST + P.GL_N] = [100, 40, 20, 4, 8, 0, 12, 16, 4, 60, 4]   # 4 iterations
    cyc[2, P.GL_FIRST + P.GL_N: P.GL_FIRST + 2 * P.GL_N] = [50, 20, 10, 2, 4, 0, 6, 8, 2, 30, 2]
    t = P.phase_table(cyc)
    s1, s2 = t["stage1"], t["stage2"]
    assert s1["problems"] == 2 and s1["iterations"]["median"] == 4
    assert s1["eval"]["median"] == 10 and s1["wait"]["median"] == 100 and s1["inv6"]["median"] == 60
    assert s1["per_iteration_total"]["median"] == (100 + 40 + 20 + 4 + 8 + 12 + 16 + 4 + 60) / 4
    assert s2["problems"] == 1 and s2["fold"]["median"] == 5


def test_k2_table(capsys):
    cyc = np.zeros((4, 32), np.int64)
    cyc[0, :8] = [10, 20, 300, 40, 5, 60, 7, 30]
    cyc[2, :8] = [30, 40, 500, 80, 15, 100, 9, 50]
    cyc[3, P.GL_FIRST + P.GL_N - 1] = 4               # a streamed pair: its K2 slots stay zero
    t = P.k2_table(cyc)
    assert t["pairs"] == 2 and list(t)[1:] == P.K2_PHASES
    assert t["gn_eval"]["median"] == 400 and t["sort_mad"]["median"] == 40 and t["match_finalize"]["p90"] == 28
    P.print_k2_table(t, None)
    out = capsys.readouterr().out
    assert "K2: 2 pairs" in out and all(n in out for n in P.K2_PHASES)
    assert P.k2_table(np.zeros((2, 32), np.int64)) == {"pairs": 0}


def test_pass_report():
    def k(name, stream, a, b):
        return {"name": name, "stream": stream, "ts": a, "end": b}
    ks = [k("void tc_hamming_kernel<1>(x)", 1, 0, 100), k("tc_hamming_kernel", 2, 90, 200), k("tc_resolve_kernel", 1, 200, 220),
          k("stream_prepare_kernel", 1, 220, 260), k("gn_loop_stream_kernel<false>", 1, 260, 300),
          k("gn_loop_stream_kernel<false>", 2, 280, 320),
          k("tc_hamming_kernel", 1, 2000, 2100)]
    passes = P.split_passes(ks)
    assert [len(p) for p in passes] == [6, 1]
    r = P.pass_report(passes[0])
    assert r["span_us"] == 320 and r["last_matcher_end_us"] == 220
    assert r["solver_after_matcher_us"] == 100 and r["gn_starts_after_last_matcher"]
    assert [e["kernel"] for e in r["streams"]["1"]] == ["tc_hamming_kernel", "tc_resolve_kernel", "stream_prepare_kernel",
                                                        "gn_loop_stream_kernel"]
