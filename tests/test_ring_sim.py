"""The callers' side of the single-request ring (csrc/agr_ring.hpp — the code the library ships) against a stand-in for the
dispatcher and the service kernel, on the CPU (tests/ring_sim.cpp).  The protocol properties the GPU tests can only show
indirectly: every operation is answered exactly once from its own payload, and callers that together hold MORE uncollected tickets
than the ring has slots finish instead of waiting for each other (AGR_EAGAIN + no-op slots)."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ring_sim(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ring") / "ring_sim")
    res = subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "ring_sim.cpp")],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    return exe


@pytest.mark.parametrize("args", [
    ("2", "0", "0", "20000"),                 # blocking callers only
    ("0", "4", "512", "100000"),              # ticket callers, well inside the ring
    ("0", "8", "4096", "40000", "20"),        # 8 x 4096 parked tickets against 16384 slots, 20 us of "GPU" per batch
    ("0", "12", "2048", "30000", "50"),       # 12 x 2048
    ("2", "6", "4096", "30000", "3"),         # blocking and ticket callers on one ring, oversubscribed
])
def test_ring_protocol_on_cpu(ring_sim, args):
    res = subprocess.run([ring_sim, *args], capture_output=True, text=True, timeout=300)      # a deadlock shows up as the timeout
    d = json.loads(res.stdout.strip().splitlines()[-1])
    assert res.returncode == 0 and d["ok"] and d["wrong_answers"] == 0 and d["served"] == d["operations"], d
    if int(args[1]) * int(args[2]) > 16384:
        assert d["eagain"] > 0 and d["skipped_slots"] >= d["eagain"], d      # the oversubscribed runs really went through the no-op path


@pytest.mark.parametrize("base", [2**48 - 40000, 2**48 - 1, 2**49 + 2**48 - 3000, 2**52 - 2**48 // 2 - 17])
def test_answers_name_full_rows_past_2_48(ring_sim, base):
    """A record's answer carries 48 bits of its row; svc_try rebuilds the rest from the rows handed out so far.  The stand-in hands
    out row base + slot number, so the rows of these runs cross a multiple of 2^48; every caller checks the full row it got."""
    for args in (("1", "3", "512", "20000", "0", str(base)), ("1", "8", "4096", "6000", "20", str(base))):
        res = subprocess.run([ring_sim, *args], capture_output=True, text=True, timeout=300)
        d = json.loads(res.stdout.strip().splitlines()[-1])
        assert res.returncode == 0 and d["ok"] and d["wrong_rows"] == 0, (d, res.stderr[-1000:])
        assert d["row_base"] == base and d["last_row"] >= base + d["operations"] - 1
        if base % 2**48 > 2**48 - 40000:
            assert d["last_row"] // 2**48 > base // 2**48          # the run really crossed the edge


def test_ring_protocol_under_thread_sanitizer(tmp_path):
    """The same simulation built with -fsanitize=thread: the shipped caller-side code (acquire / release accesses on the answer
    cells, release / acquire on the ready words, streaming stores behind an sfence) has no data race ThreadSanitizer can see."""
    exe = str(tmp_path / "ring_sim_tsan")
    res = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-o", exe, os.path.join(ROOT, "tests", "ring_sim.cpp")],
                         capture_output=True, text=True, timeout=300)
    if res.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime in this image: " + res.stderr[-200:])
    assert "-Wtsan" not in res.stderr                       # (atomic_thread_fence is not modelled by TSAN: the header must not need it)
    for args in (("1", "3", "512", "10000"), ("0", "8", "4096", "6000", "20")):
        run = subprocess.run([exe, *args], capture_output=True, text=True, timeout=600)
        assert "ThreadSanitizer" not in run.stderr, run.stderr[-2000:]
        d = json.loads(run.stdout.strip().splitlines()[-1])
        assert run.returncode == 0 and d["ok"], d
