"""Variable-length records (AGR_CFG_VARLEN, BASELINE config 5: 128 B - 4 KB bodies) through the byte-tiled K1 kernel:
parity with the (size-agnostic) Python oracle, stored bytes round trip, checksum, tile-ownership edge cases."""
import dataclasses

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from kats import SCENARIOS, load_golden
from scenario import run_oracle, run_engine, assert_same, random_scenario, Req, rid_of, make_var_batch

pytestmark = pytest.mark.gpu
GOLD, _ = load_golden()
VAR = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN
FORMS = {"staged": 0, "lsu": 0x20}      # k1_variant: K1v through per-warp TMA stages / its LSU form (bit 0x20)


def engine(flags=VAR, form="staged", **kw):
    kw.setdefault("slab_rows", 1 << 15)
    kw.setdefault("max_agents", 256)
    kw.setdefault("vslab_bytes", 256 << 20)
    return A.Engine(flags=flags, k1_variant=FORMS[form], **kw)


def with_bodies(events, seed):
    """log-uniform body sizes in [128 B, 4 KB] (BASELINE config 5)"""
    rng = np.random.default_rng(seed)
    out = []
    for e in events:
        if e[0] == "req":
            n = int(np.exp(rng.uniform(np.log(128), np.log(4096))))
            out.append(("req", dataclasses.replace(e[1], body=rng.integers(32, 127, n, dtype=np.uint8).tobytes()), e[2]))
        else:
            out.append(e)
    return out


@pytest.mark.parametrize("kat", sorted(SCENARIOS))
@pytest.mark.parametrize("flags", [VAR, VAR | K.AGR_CFG_MINT_IDS])
@pytest.mark.parametrize("form", FORMS)
def test_kats_variable_length(form, kat, flags):
    ev = with_bodies(SCENARIOS[kat], 1)
    with engine(flags, form) as eng:
        got = run_engine(eng, ev)
    exp = GOLD[kat]
    assert got.verdicts == exp["verdicts"] and got.ticks == exp["ticks"] and got.records == exp["records"]
    for a, qs in exp["lists"].items():
        assert got.lists[a] == qs, (kat, a)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("form", FORMS)
def test_random_streams_variable_length(form, seed):
    ev = with_bodies(random_scenario(300 + seed, n_events=500, n_agents=2 + seed % 5, p_replay=0.15), seed)
    ref = run_oracle(ev)
    with engine(VAR | (K.AGR_CFG_MINT_IDS if seed % 2 else 0), form) as eng:
        assert_same(ref, run_engine(eng, ev, rng=np.random.default_rng(seed)))


def test_stored_bytes_checksum_and_tile_edges():
    """Record sizes chosen to hit the byte-tile machinery: records that end exactly on an 8 KiB tile boundary, the
    longest legal record (8192 B), runs of minimum-size records (96 B header + 16 B), tiles in which no record starts.
    Both forms of K1v, one after the other."""
    for form in FORMS:
        stored_bytes_checksum_and_tile_edges(form)


def stored_bytes_checksum_and_tile_edges(form):
    sizes = [8192 - 96 - 48] * 3 + [16] * 200 + [4000, 8192 - 96 - 48, 16, 8192 - 96 - 48, 8192 - 96 - 48] + [100, 3000, 5, 0, 777] * 40
    rng = np.random.default_rng(3)
    reqs = []
    for i, n in enumerate(sizes):
        hdr_path = len(f"/agent/agent-1/c") + len("A: b\n")
        body = rng.integers(0, 256, max(0, n - 0), dtype=np.uint8).tobytes()
        reqs.append(Req("agent-1" if i % 3 else "agent-2", rid_of(i + 1), i + 1, subpath="/c", body=body, headers={"A": "b"}))
    blob, offs = make_var_batch(reqs)
    lens = np.diff(offs)
    assert lens.max() <= K.AGR_VAR_MAX_RECORD and (lens % 16 == 0).all()
    with engine(form=form, slab_rows=1 << 12) as eng:
        eng.set_agent_state("agent-1", "stopped"); eng.set_agent_state("agent-2", "running")
        # two batches: the second starts at an arbitrary (16 B aligned) slab offset
        cut = 150
        v1, ids1, f1 = eng.ingest_var(np.ascontiguousarray(blob[: offs[cut]]), offs[: cut + 1].copy())
        v2, ids2, f2 = eng.ingest_var(np.ascontiguousarray(blob[offs[cut]:]), (offs[cut:] - offs[cut]).astype(np.uint32))
        v = np.concatenate([v1, v2])
        exp_code = [K.AGR_V_QUEUED if i % 3 else K.AGR_V_FORWARD for i in range(len(reqs))]
        assert [int(x) for x in v["code"]] == exp_code and f1 == 0 and f2 == cut
        # checksum = position-weighted sums over the stored bytes of each record
        ck = eng.debug_read("cksum", 0, len(reqs))
        for i in (0, 1, 2, 3, 150, 203, 204, 205, 206, 207, len(reqs) - 1):
            w = blob[offs[i]: offs[i + 1]].view(np.uint32).astype(np.uint64)
            c0 = int(w.sum()) & 0xFFFFFFFF
            c1 = int((w * np.arange(1, len(w) + 1, dtype=np.uint64)).sum()) & 0xFFFFFFFF
            assert int(ck[i]) == (c1 << 32) | c0, i
        # stored bytes come back exactly (status bytes aside), by id and through the replay scan
        for i in (0, 2, 3, 150, 206, len(reqs) - 1):
            raw = eng.get_record_var(reqs[i].agent_id, reqs[i].rid)
            src = blob[offs[i]: offs[i + 1]]
            assert len(raw) == len(src) and raw[96:].tobytes() == src[96:].tobytes() and raw[:84].tobytes() == src[:84].tobytes()
        eng.set_agent_state("agent-1", "running")
        disp, vblob, voffs = eng.replay_scan_var()
        # agent-1's queued records, then agent-2's forwarded-but-unanswered ones (still pending: Q1 / Q16), FIFO inside each
        exp_idx = [i for i in range(len(reqs)) if i % 3] + [i for i in range(len(reqs)) if i % 3 == 0]
        assert [bytes(d["request_id"]) for d in disp] == [reqs[i].rid for i in exp_idx]
        for j in (0, 1, len(exp_idx) // 2, len(exp_idx) - 1):
            i = exp_idx[j]
            assert vblob[int(voffs[j]) + 96: int(voffs[j + 1])].tobytes() == blob[offs[i] + 96: offs[i + 1]].tobytes()


def test_bad_wire_shapes_are_rejected():
    with engine(slab_rows=1 << 10) as eng:
        eng.set_agent_state("agent-1", "running")
        blob, offs = make_var_batch([Req("agent-1", rid_of(1), 1)])
        bad = offs.copy(); bad[1] -= 8
        with pytest.raises(A.AgrError):
            eng.ingest_var(blob, bad)                              # not a multiple of 16
        with pytest.raises(A.AgrError):
            eng.ingest_var(np.zeros(16384, dtype=np.uint8), np.array([0, 16384], dtype=np.uint32))   # longer than 8192
        with pytest.raises(A.AgrError):
            eng.ingest(np.zeros(1, dtype=A.record_dtype))          # fixed-stride call on a variable-length engine
