"""The single-request ring of a variable-length engine (AGR_CFG_COMBINE | AGR_CFG_VARLEN), on the CPU against
tests/ring_sim_var.cpp's stand-in for the dispatcher and the service kernel: records are spans of 1 .. 16 slots mixed with
outcome spans, every operation is answered exactly once from a checksum of all the bytes its caller wrote read across the span,
the record bytes a batch takes are summed by the scan and stay within the byte budget, spans cross the ring's end, and callers
that hold more tickets than the ring has slots get AGR_EAGAIN instead of waiting."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "ring_sim_var.cpp")
RUNS = [
    ("2", "0", "0", "20000", "0"),                  # blocking callers: record spans, outcome spans, plain outcomes
    ("0", "4", "512", "30000", "0"),                # ticket callers
    ("0", "8", "4096", "10000", "20"),              # oversubscribed: AGR_EAGAIN + no-op spans while continuations are in flight
    ("2", "6", "4096", "10000", "3", "12288"),      # a byte budget below a batch's stage: batches end early, a lone 8 KiB
                                                    # record still goes
]


@pytest.fixture(scope="module")
def ring_sim(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ring_var") / "ring_sim_var")
    res = subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-Wall", "-o", exe, SRC], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    return exe


def check(d, args):
    assert d["ok"] and d["wrong_answers"] == 0 and d["served"] == d["operations"], d
    assert d["operations"] == (int(args[0]) + int(args[1])) * int(args[3]), d
    assert 0 < d["max_staged"] <= 128, d
    assert d["record_spans"] > 0 and d["span_slots"] > d["record_spans"], d
    assert d["capped_headers"] > 0, d


@pytest.mark.parametrize("args", RUNS)
def test_record_spans_on_cpu(ring_sim, args):
    res = subprocess.run([ring_sim, *args], capture_output=True, text=True, timeout=300)
    d = json.loads(res.stdout.strip().splitlines()[-1])
    assert res.returncode == 0, d
    check(d, args)
    assert d["max_record_slots"] == 16 and d["wrapped_spans"] > 0, d
    if int(args[1]) * int(args[2]) > 16384:
        assert d["eagain"] > 0 and d["skipped_slots"] > 0, d
    if len(args) > 5:
        assert d["max_batch_bytes"] <= max(int(args[5]), 8192), d


def test_record_spans_under_thread_sanitizer(tmp_path):
    exe = str(tmp_path / "ring_sim_var_tsan")
    res = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-o", exe, SRC],
                         capture_output=True, text=True, timeout=300)
    if res.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime in this image: " + res.stderr[-200:])
    for args in (("1", "3", "512", "3000", "0"), ("0", "8", "4096", "2000", "20", "8192")):
        run = subprocess.run([exe, *args], capture_output=True, text=True, timeout=600)
        assert "ThreadSanitizer" not in run.stderr, run.stderr[-2000:]
        d = json.loads(run.stdout.strip().splitlines()[-1])
        assert run.returncode == 0, d
        check(d, args)
