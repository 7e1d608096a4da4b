"""The byte layout of a snapshot file: header, agent table, then every section in order, sized from the header alone.  A
round trip (tests/test_durability_gpu.py) cannot see a section that snapshot and restore both move or resize the same way;
this test reads the file itself and checks each section against what the engine reports for the same rows."""
import ctypes as C

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from jsoncase import make_requests, records_array, var_batch
from snapfile import parse

pytestmark = pytest.mark.gpu

SLAB_ROWS = 1 << 12
RING_ROWS, RESP, VSLAB = 512, 64 << 10, 1 << 20     # ring modes: small enough that rows and bytes go round within a few batches
SEC = 1_000_000_000
T0, STEP = 1_700_000_000 * SEC, 3600 * SEC
SECRET = 0x5EED_1234_ABCD_0001
AGENTS = ["agent-1700000000000000001", "agent-1700000000000000002", "agent-1700000000000000003", "agent-1700000000000000004"]
STATUS = ["running", "running", "stopped", "running"]
MODES = {"hash": K.AGR_CFG_PERSISTENCE, "mint": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS,
         "var": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN | K.AGR_CFG_MINT_IDS,
         "ring": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING,
         "var_ring": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING}

AGENT_ENTRY = 32 + 1                      # NUL-padded agent id, status byte


def device_bytes(ptr: int, n: int) -> bytes:
    out = np.zeros(max(n, 1), dtype=np.uint8)
    assert C.CDLL("libcudart.so").cudaMemcpy(C.c_void_p(out.ctypes.data), C.c_void_p(ptr), C.c_size_t(n), 2) == 0
    return out[:n].tobytes()


def outcomes(rows):
    outs = np.zeros(len(rows), dtype=A.outcome_dtype)
    for j, (rid, agent, kind, http, seq) in enumerate(rows):
        outs[j]["request_id"] = np.frombuffer(rid, dtype=np.uint8)
        outs[j]["agent_id"] = agent.encode()
        outs[j]["kind"], outs[j]["http_status"], outs[j]["seq"] = kind, http, seq
    return outs


@pytest.mark.parametrize("mode", sorted(MODES))
def test_snapshot_sections_match_the_engine(mode, tmp_path):
    flags = MODES[mode]
    var, ring = bool(flags & K.AGR_CFG_VARLEN), bool(flags & K.AGR_CFG_RING)
    S = RING_ROWS if ring else SLAB_ROWS
    kw = dict(slab_rows=S, max_agents=16, flags=flags, id_secret=SECRET, vslab_bytes=VSLAB if ring else 8 << 20,
              resp_bytes=RESP if ring else 0)
    rng = np.random.default_rng(11)
    with A.Engine(**kw) as eng:
        for a, s in zip(AGENTS, STATUS):
            eng.set_agent_state(a, s)
        reqs, ids, var_lens, want, applied = {}, {}, {}, {}, set()    # by logical row
        blob_total = resp_total = 0
        for rnd in range(40):
            # append-only: two batches, the second behind the first.  Ring: until the rows, the response bytes and the record
            # bytes have each gone round at least once, expiring and releasing everything older than the previous round
            if rnd == 2 and not ring:
                break
            if ring and eng.stats()["rows_used"] > S and resp_total > RESP and (blob_total > VSLAB or not var):
                break
            now = T0 + rnd * STEP
            if ring and rnd:
                eng.expire(now, STEP + STEP // 2)
                eng.reclaim()
            batch = make_requests(50 + rnd, 160, AGENTS, max_payload=1000 if var else 416, big_bodies=var)
            for k, r in enumerate(batch):
                r.now = now + k * SEC
            if var:
                blob, offs = var_batch(batch)
                _, got, first = eng.ingest_var(blob, offs)
                blob_total += int(offs[-1])
                var_lens.update((first + k, int(x)) for k, x in enumerate(np.diff(offs)))
            else:
                got = np.zeros((len(batch), 16), dtype=np.uint8)
                first = eng.ingest_ex(records_array(batch), np.zeros(len(batch), dtype=A.verdict_dtype), got)
            for k, (r, x) in enumerate(zip(batch, got)):
                reqs[first + k] = r
                ids[first + k] = bytes(x) if flags & K.AGR_CFG_MINT_IDS else r.rid
            # responses with headers and body, and transitions without bytes; then error texts, three rounds, so that the
            # records run out of retries (max_retries 3) and land in the failed log
            t = now + 600 * SEC
            ops, segs, hlens, failing = [], [], [], []
            for j, k in enumerate(rng.permutation(len(batch))[:100]):
                row, r = first + int(k), batch[int(k)]
                if j % 3 == 0:
                    failing.append(row)
                elif j % 7 == 1:
                    ops.append((row, (ids[row], r.agent_id, K.AGR_OUT_DIAL_ERR, 0, t))); segs.append(b""); hlens.append(0)
                else:
                    hdr = b"Content-Type: text/plain\n" if j % 2 else b""
                    body = bytes(rng.integers(0, 256, int(rng.integers(0, 120 if ring else 300)), dtype=np.uint8))
                    ops.append((row, (ids[row], r.agent_id, K.AGR_OUT_RESPONSE, 200, t))); segs.append(hdr + body); hlens.append(len(hdr))
                    want[row] = ("resp", hdr, body)
            rc, res = eng.complete_ex(outcomes([o for _, o in ops]), segs, np.array(hlens, dtype=np.uint32))
            assert rc == 0
            resp_total += sum((len(x) + 15) // 16 * 16 for x in segs)
            applied |= {row for (row, _), x in zip(ops, res) if x == 0}
            for _ in range(3):
                texts = [bytes(rng.integers(0, 256, int(rng.integers(1, 60)), dtype=np.uint8)) for _ in failing]
                rc, res = eng.complete_ex(outcomes([(ids[i], reqs[i].agent_id, K.AGR_OUT_ERROR, 0, t) for i in failing]), texts)
                assert rc == 0
                resp_total += sum((len(x) + 15) // 16 * 16 for x in texts)
                for i, x, y in zip(failing, texts, res):
                    want[i] = ("err", x)
                    if y == 0:
                        applied.add(i)
                    else:
                        applied.discard(i)
        st = eng.stats()
        path = str(tmp_path / f"{mode}.snap")
        eng.snapshot(path)
        data = open(path, "rb").read()
        hd, agents, sec = parse(data)                         # (parse asserts that the sections account for every byte of the file)

        assert hd["magic"] == b"AGRSNAP3"
        assert int(hd["flags"]) == flags & (K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_VARLEN | K.AGR_CFG_RING)
        assert int(hd["id_secret"]) == SECRET and int(hd["slab_rows"]) == S
        used, tail = int(hd["rows_used"]), int(hd["tail"])
        assert used == st["rows_used"] and tail == st["rows_tail"]
        entries = [agents[at: at + AGENT_ENTRY] for at in range(0, len(agents), AGENT_ENTRY)]
        assert [(e[:32].rstrip(b"\0").decode(), e[32]) for e in entries] == [(a, K.AGENT_STATUS_CODES[s]) for a, s in zip(AGENTS, STATUS)]
        if ring:                                              # each ring has gone round: its sections hold one lap
            assert used > S and tail > 0 and int(hd["resp_used"]) > int(hd["resp_cap"]) == RESP
            assert not var or int(hd["vused"]) > int(hd["vcap"]) == VSLAB
        rows = min(used, S)
        phys = (lambda L: L % S) if ring else (lambda L: L)

        # per-row sections are physical rows 0..rows-1; read the same rows through their logical numbers
        lo = used - rows
        for name in ("state", "route", "aux", "cksum", "mtime"):
            assert np.array_equal(sec[name], np.roll(eng.debug_read(name, lo, rows), lo % S)), name
        slab_base = eng.slab_ptr(tail) - phys(tail) * 512
        assert sec["slab"].tobytes() == device_bytes(slab_base, len(sec["slab"]))
        live = [L for L in range(tail, used) if L in reqs]
        if var:
            for L in live:
                p = phys(L)
                assert int(sec["vlen"][p]) == var_lens[L] and int(sec["voff"][p]) + var_lens[L] <= len(sec["slab"])
            if not ring:
                lens = [var_lens[L] for L in range(used)]
                assert sec["voff"].tolist() == np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
        else:
            assert len(sec["slab"]) == rows * 512

        assert len(sec["completed_log"]) == st["completed_log_len"] > 0
        assert len(sec["failed_log"]) == st["failed_log_len"] > 0
        stored = 0
        for L in applied & set(want) & set(live):
            w, p = want[L], phys(L)
            if w[0] == "resp":
                o, n = int(sec["resp_off"][p]), int(sec["resp_len"][p])
                assert (sec["resp"][o: o + n].tobytes(), int(sec["resp_hlen"][p])) == (w[1] + w[2], len(w[1]))
            else:
                o, n = int(sec["err_off"][p]), int(sec["err_len"][p])
                assert sec["resp"][o: o + n].tobytes() == w[1]
            stored += 1
        assert stored > 100
