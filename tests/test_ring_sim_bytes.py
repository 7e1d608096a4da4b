"""The single-request ring with outcomes that carry their bytes inline (SVC_OP_OUTCOME_BYTES, agr_submit_complete_ex), on the
CPU against tests/ring_sim_bytes.cpp's stand-in for the dispatcher and the service kernel: every operation is answered exactly
once, from a checksum of the very bytes its caller wrote, and no batch holds more than 128 records plus such outcomes (each
takes a whole 512 B slot of the kernel's stage)."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "ring_sim_bytes.cpp")
RUNS = [
    ("2", "0", "0", "20000", "0"),          # blocking callers: plain outcomes and outcomes with bytes alternate
    ("0", "4", "512", "60000", "0"),        # ticket callers: records and outcomes with bytes
    ("0", "8", "4096", "30000", "20"),      # oversubscribed: AGR_EAGAIN + no-op slots with bytes in flight
    ("2", "6", "4096", "20000", "3"),
]


@pytest.fixture(scope="module")
def ring_sim(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ring_bytes") / "ring_sim_bytes")
    res = subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-Wall", "-o", exe, SRC], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    return exe


@pytest.mark.parametrize("args", RUNS)
def test_outcomes_with_bytes_on_cpu(ring_sim, args):
    res = subprocess.run([ring_sim, *args], capture_output=True, text=True, timeout=300)
    d = json.loads(res.stdout.strip().splitlines()[-1])
    assert res.returncode == 0 and d["ok"] and d["wrong_answers"] == 0 and d["served"] == d["operations"], d
    if int(args[1]) * int(args[2]) > 16384:
        assert d["eagain"] > 0, d


def test_outcomes_with_bytes_under_thread_sanitizer(tmp_path):
    exe = str(tmp_path / "ring_sim_bytes_tsan")
    res = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-o", exe, SRC],
                         capture_output=True, text=True, timeout=300)
    if res.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime in this image: " + res.stderr[-200:])
    for args in (("1", "3", "512", "8000", "0"), ("0", "8", "4096", "5000", "20")):
        run = subprocess.run([exe, *args], capture_output=True, text=True, timeout=600)
        assert "ThreadSanitizer" not in run.stderr, run.stderr[-2000:]
        d = json.loads(run.stdout.strip().splitlines()[-1])
        assert run.returncode == 0 and d["ok"], d
