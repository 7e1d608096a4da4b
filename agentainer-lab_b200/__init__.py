"""agentainer-lab_b200 — H100-native (sm_90a CUDA) request queue / replay / route engine for Agentainer's
/agent/<id>/ hot path.  The product is the C-ABI shared library built from csrc/ (include/agentainer_gpu.h);
this Python package is only the thin ctypes mirror used by tests and bench.py, plus the build helper.

There is no CPU fallback: importing works anywhere (so the ABI can be checked without a GPU), but creating an
Engine without an sm_90 device raises."""
from .build import build_native, build_host, lib_path   # noqa: F401
from .binding import (                              # noqa: F401
    Engine, AgrError, load_library, record_dtype, header_dtype, outcome_dtype, verdict_dtype, dispatch_dtype,
    synth_fill_host, synth_agent_id, var_record_len, agent_hash, agent_shard, comm_unique_id, json_decode, ABI_SYMBOLS,
)
from . import constants                             # noqa: F401
