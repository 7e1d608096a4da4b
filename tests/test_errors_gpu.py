"""Error behaviour of the C-ABI on a live engine: capacities, argument checks, 'log and continue' result codes."""
import ctypes as C

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from scenario import Req, rid_of, make_records

pytestmark = pytest.mark.gpu


def test_capacities_and_argument_checks():
    with A.Engine(slab_rows=256, max_agents=4, max_batch=128) as eng:
        lib = eng.lib
        for k in range(4):
            assert eng.set_agent_state(f"agent-{k}", "running") == k
        with pytest.raises(A.AgrError) as e:
            eng.set_agent_state("agent-4", "running")                       # agent table full
        assert e.value.code == K.AGR_ENOSPC
        with pytest.raises(A.AgrError) as e:
            eng.set_agent_state("a" * 32, "running")                        # id must fit 31 bytes + NUL
        assert e.value.code == K.AGR_EINVAL
        assert eng.set_agent_state("agent-0", "stopped") == 0                # updating an existing agent still works
        recs = make_records([Req("agent-1", rid_of(i), i) for i in range(1, 201)])
        with pytest.raises(A.AgrError) as e:
            eng.ingest(recs)                                                 # n > max_batch
        assert e.value.code == K.AGR_EINVAL
        v, first = eng.ingest(np.ascontiguousarray(recs[:128]))
        assert first == 0 and (v["code"] == K.AGR_V_FORWARD).all()
        v, first = eng.ingest(np.ascontiguousarray(recs[128:200]))
        assert first == 128
        with pytest.raises(A.AgrError) as e:
            eng.ingest(make_records([Req("agent-1", rid_of(1000 + i), i) for i in range(100)]))   # 200 + 100 > 256 rows
        assert e.value.code == K.AGR_ENOSPC
        s = eng.stats()
        assert s["rows_used"] == 200 and s["stored"] == 200                 # the refused batch left no trace
        # output array too small: AGR_ECAP and the needed count
        n = C.c_uint32()
        out = np.zeros(10, dtype=A.record_dtype)
        rc = lib.agr_pending(eng.h, b"agent-1", C.c_void_p(out.ctypes.data), 10, C.byref(n))
        assert rc == K.AGR_ECAP and n.value == 200
        assert lib.agr_strerror(rc) == b"output array too small"
        # per-outcome results: unknown id / unknown agent / wrong agent are misses, the batch still succeeds (Q20)
        outs = np.zeros(4, dtype=A.outcome_dtype)
        outs["kind"], outs["http_status"] = K.AGR_OUT_RESPONSE, 200
        outs[0]["request_id"], outs[0]["agent_id"] = np.frombuffer(rid_of(5), dtype=np.uint8), b"agent-1"
        outs[1]["request_id"], outs[1]["agent_id"] = np.frombuffer(rid_of(5), dtype=np.uint8), b"agent-2"     # wrong agent
        outs[2]["request_id"], outs[2]["agent_id"] = np.frombuffer(rid_of(999), dtype=np.uint8), b"agent-1"   # unknown id
        outs[3]["request_id"], outs[3]["agent_id"] = np.frombuffer(rid_of(6), dtype=np.uint8), b"agent-nope"  # unknown agent
        assert list(eng.complete(outs)) == [0, K.AGR_ENOTFOUND, K.AGR_ENOTFOUND, K.AGR_ENOTFOUND]
        assert eng.stats()["completion_misses"] == 3
        # zero-length calls are no-ops
        assert eng.ingest(np.zeros(0, dtype=A.record_dtype))[0].shape == (0,)
        assert eng.complete(np.zeros(0, dtype=A.outcome_dtype)).shape == (0,)


def test_bad_configs_are_rejected():
    retired_k1 = [dict(slab_rows=1 << 10, k1_variant=v) for v in (1, 5, 0x10, 0x100)]     # K1 alternates that no longer exist
    for kw in [dict(slab_rows=1 << 10, table_slots=1000), dict(slab_rows=1 << 10, table_slots=1024), dict(slab_rows=1 << 31)] + retired_k1:
        with pytest.raises(A.AgrError) as e:
            A.Engine(**kw)
        assert e.value.code == K.AGR_EINVAL
    with pytest.raises(A.AgrError) as e:
        A.Engine(device=63, slab_rows=1 << 10)
    assert e.value.code == K.AGR_ENODEV


def test_sharded_calls_need_a_communicator():
    with A.Engine(slab_rows=1 << 10) as eng:
        with pytest.raises(A.AgrError) as e:
            eng.ingest_sharded(np.zeros(1, dtype=A.record_dtype))
        assert e.value.code == K.AGR_ECOMM


def test_bulk_agent_state_feed():
    """agr_set_agent_states == the same agr_set_agent_state calls one by one (small and table-upload paths)."""
    import numpy as np
    from jsoncase import make_requests, records_array
    names = [f"agent-17000000000000{i:05d}" for i in range(300)]
    with A.Engine(slab_rows=1 << 12, max_agents=512) as one, A.Engine(slab_rows=1 << 12, max_agents=512) as bulk:
        sts = ["running" if i % 3 else "stopped" for i in range(300)]
        for n_, s_ in zip(names, sts):
            one.set_agent_state(n_, s_)
        assert list(bulk.set_agent_states(names[:5], sts[:5])) == [0, 1, 2, 3, 4]            # per-entry copies
        assert list(bulk.set_agent_states(names, sts)) == list(range(300))                    # table upload
        flip = ["stopped" if s == "running" else "running" for s in sts]
        for n_, s_ in zip(names[::7], flip[::7]):
            one.set_agent_state(n_, s_)
        bulk.set_agent_states(names[::7], flip[::7])
        reqs = make_requests(4, 600, names)
        recs = records_array(reqs)
        outs = []
        for eng in (one, bulk):
            out = np.zeros(600, dtype=A.verdict_dtype); ids = np.zeros((600, 16), dtype=np.uint8)
            eng.ingest_ex(recs, out, ids)
            outs.append(out.copy())
        assert (outs[0] == outs[1]).all() and len(set(outs[0]["code"].tolist())) >= 2
        bad = bulk.lib.agr_set_agent_states(bulk.h, None, None, 3, None)
        assert bad == K.AGR_EINVAL
