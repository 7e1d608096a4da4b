"""SURVEY 8f-2: snapshot / restore (what Redis persistence gave the reference) and the integrity sweep."""
import os

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from scenario import run_oracle, run_engine, assert_same, random_scenario

pytestmark = pytest.mark.gpu
MODES = {"hash": K.AGR_CFG_PERSISTENCE, "mint": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS,
         "var": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN | K.AGR_CFG_MINT_IDS}


class Restarting:
    """An engine that is snapshotted, destroyed and restored from the file in the middle of a stream: to the scenario
    driver it is one engine; every call after the restart goes to the restored one."""

    def __init__(self, flags, path, restart_after_calls):
        self.kw = dict(slab_rows=1 << 15, max_agents=256, flags=flags, vslab_bytes=64 << 20)
        self.eng, self.path, self.left = A.Engine(**self.kw), path, restart_after_calls
        self.mint, self.varlen = self.eng.mint, self.eng.varlen
        self.restarts = 0

    def __getattr__(self, name):
        target = getattr(self.eng, name)
        if name in ("ingest", "ingest_var", "complete") and self.left is not None:
            self.left -= 1
            if self.left == 0:
                self.left = None
                self.eng.snapshot(self.path)
                self.eng.close()                                   # "server restart"
                self.eng = A.Engine(restore_from=self.path, **self.kw)
                self.restarts += 1
                target = getattr(self.eng, name)
        return target

    def close(self):
        self.eng.close()


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("online", [False, True], ids=["blocking", "online"])
def test_restart_in_mid_stream_is_invisible(mode, seed, online, tmp_path):
    ev = random_scenario(400 + seed, n_events=500, n_agents=5, p_replay=0.15)
    if mode == "var":
        from test_varlen_gpu import with_bodies
        ev = with_bodies(ev, seed)
    ref = run_oracle(ev)
    flags = MODES[mode] | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0)
    r = Restarting(flags, str(tmp_path / "agr.snap"), restart_after_calls=12 + seed)
    try:
        got = run_engine(r, ev, max_batch=40)
        assert r.restarts == 1
        assert_same(ref, got)
        rows, bad = r.eng.verify()
        assert rows > 100 and bad == 0
    finally:
        r.close()


@pytest.mark.parametrize("online", [False, True], ids=["blocking", "online"])
def test_a_failed_flush_fails_the_snapshot(online):
    """The file of a small engine fits stdio's buffer whole, so its bytes reach the device only when the file is closed:
    /dev/full takes every write and refuses that flush.  The snapshot must report it, not succeed."""
    from scenario import Req, rid_of, make_records
    flags = MODES["mint"] | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0)
    with A.Engine(slab_rows=1 << 10, max_agents=16, flags=flags) as eng:
        eng.set_agent_state("agent-1", "running")
        eng.ingest(make_records([Req("agent-1", rid_of(i), i) for i in range(1, 5)]))   # 4 rows: ~2.5 KiB of file
        with pytest.raises(A.AgrError) as e:
            eng.snapshot("/dev/full")
        assert e.value.code == K.AGR_EINVAL


def test_verify_detects_a_flipped_bit(tmp_path):
    import ctypes as C
    recs = A.synth_fill_host(0, 5000, seed=8, n_agents=4)
    with A.Engine(slab_rows=1 << 13, max_agents=16) as eng:
        for k in range(4):
            eng.set_agent_state(A.synth_agent_id(k), "stopped")
        eng.ingest(recs)
        assert eng.verify() == (5000, 0)
        # corrupt one byte of row 1234 directly in HBM
        one = np.array([0xA5], dtype=np.uint8)
        C.CDLL("libcudart.so").cudaMemcpy(C.c_void_p(eng.slab_ptr(1234) + 300), C.c_void_p(one.ctypes.data), C.c_size_t(1), 1)
        assert eng.verify() == (5000, 1)
        eng.snapshot(str(tmp_path / "bad.snap"))
    with A.Engine(slab_rows=1 << 13, max_agents=16, restore_from=str(tmp_path / "bad.snap")) as eng2:
        assert eng2.verify() == (5000, 1)                          # the snapshot carries the checksums: corruption is still seen
        assert [bytes(x) for x in eng2.list(A.synth_agent_id(0), 0)] == [bytes(x) for x in recs["request_id"][recs["agent_id"] == A.synth_agent_id(0).encode()]]


def test_restore_rejects_mismatched_mode(tmp_path):
    p = str(tmp_path / "m.snap")
    with A.Engine(slab_rows=1 << 10, flags=MODES["mint"]) as eng:
        eng.set_agent_state("agent-1", "running")
        eng.snapshot(p)
    with pytest.raises(A.AgrError):
        A.Engine(slab_rows=1 << 10, flags=MODES["hash"], restore_from=p)
    with pytest.raises(A.AgrError):
        A.Engine(slab_rows=1 << 10, flags=MODES["mint"], id_secret=12345, restore_from=p)


def test_stored_response_bodies_round_trip_and_survive_a_restart(tmp_path):
    """StoreResponse keeps the response with the record (requests.go:142-147,165); the bytes travel off the hot path."""
    from scenario import Req, rid_of, make_records
    p = str(tmp_path / "r.snap")
    with A.Engine(slab_rows=1 << 10, max_agents=16, flags=MODES["mint"]) as eng:
        eng.set_agent_state("agent-1", "running")
        v, first = eng.ingest(make_records([Req("agent-1", rid_of(i), i) for i in range(1, 6)]))
        ids = [bytes(x) for x in eng.mint_ids(first, 5)]
        assert eng.get_response_body("agent-1", ids[0]) == b""
        assert eng.store_response_body("agent-1", ids[0], b'Content-Type: application/json\n\n{"reply":"hi"}')
        assert eng.store_response_body("agent-1", ids[3], b"x" * 5000)
        assert eng.store_response_body("agent-1", ids[0], b"second response wins")            # like the reference's SET
        assert not eng.store_response_body("agent-1", rid_of(77), b"nope")
        assert eng.get_response_body("agent-1", ids[0]) == b"second response wins"
        assert eng.get_response_body("agent-1", ids[3]) == b"x" * 5000
        assert eng.get_response_body("agent-2", ids[3]) is None
        eng.snapshot(p)
    with A.Engine(slab_rows=1 << 10, max_agents=16, flags=MODES["mint"], restore_from=p) as eng2:
        assert eng2.get_response_body("agent-1", ids[0]) == b"second response wins"
        assert eng2.get_response_body("agent-1", ids[3]) == b"x" * 5000
        assert eng2.get_response_body("agent-1", ids[1]) == b""
