"""CPU checks of the drop-in boundary: the library loads, exports every symbol include/agentainer_gpu.h declares,
struct sizes / constants agree with the header, and creation fails loudly without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.binding import AgrConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "agentainer_gpu.h")).read()


def declared_symbols():
    body = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    return sorted(set(re.findall(r"\b(agr_[a-z0-9_]+)\s*\(", body)))


def test_every_declared_symbol_is_exported(lib):
    syms = declared_symbols()
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert sorted(A.ABI_SYMBOLS) == syms
    assert len(syms) == 71 and "agr_debug_skip_arrivals" in syms and "agr_debug_k4" in syms


def test_header_constants_match_python():
    for name, val in re.findall(r"#define\s+(AGR_[A-Z0-9_]+)\s+(-?\d+|0x[0-9a-fA-F]+)u?\b", HEADER):
        if hasattr(K, name):
            assert getattr(K, name) == int(val, 0), name
    enums = re.findall(r"(AGR_[A-Z0-9_]+)\s*=\s*(\d+)", re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S))
    assert len(enums) > 20
    for name, val in enums:
        assert getattr(K, name) == int(val), name


def test_struct_sizes():
    assert A.record_dtype.itemsize == 512 and A.outcome_dtype.itemsize == 64
    assert A.verdict_dtype.itemsize == 8 and A.dispatch_dtype.itemsize == 32
    assert A.record_dtype.fields["payload"][1] == K.AGR_HEADER_BYTES
    assert A.record_dtype.fields["seq"][1] == 64 and A.record_dtype.fields["agent_id"][1] == 32
    assert C.sizeof(AgrConfig) == 72


def test_abi_version_and_strerror(lib):
    assert lib.agr_abi_version() == 2
    assert lib.agr_strerror(K.AGR_ENOTFOUND) == b"not found"
    assert lib.agr_strerror(K.AGR_ENODEV) == b"no usable CUDA device"


def test_shard_hash_is_fnv1a64():
    def fnv(s):
        h = 0xCBF29CE484222325
        for b in s.encode():
            h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
        return h
    for s in ["agent-1700000000000000000", "a", "agent-1753000000123456789"]:
        assert A.agent_hash(s) == fnv(s)
        assert A.agent_shard(s, 8) == fnv(s) % 8


def test_create_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(A.AgrError) as e:
        A.Engine(slab_rows=1024)
    assert e.value.code == K.AGR_ENODEV
    assert "no CPU fallback" in str(e.value)


def test_null_arguments_are_rejected(lib):
    n = C.c_uint32()
    assert lib.agr_ingest(None, None, 1, None, None) == K.AGR_EINVAL
    assert lib.agr_complete(None, None, 0, None) == K.AGR_EINVAL
    assert lib.agr_replay_scan(None, None, None, 0, C.byref(n)) == K.AGR_EINVAL
    assert lib.agr_create(None, None) == K.AGR_EINVAL
    assert lib.agr_debug_skip_arrivals(None, C.c_uint64(1)) == K.AGR_EINVAL
    assert lib.agr_debug_world(None, 0, 2) == K.AGR_EINVAL
    assert lib.agr_debug_exchange_end(None, None, None) == K.AGR_EINVAL


def test_ctypes_structs_match_the_c_header(tmp_path):
    """Compile a C program against include/agentainer_gpu.h that prints sizeof / offsetof of every struct the Python
    harness mirrors, and compare with ctypes and numpy: a silent drift would corrupt stats or configs."""
    import subprocess
    from agentainer_lab_b200.binding import AgrStats, AgrExchangeInfo, AgrSynth, AgrDecoded
    structs = {"agr_config": AgrConfig, "agr_stats": AgrStats, "agr_exchange_info": AgrExchangeInfo, "agr_synth": AgrSynth,
               "agr_decoded": AgrDecoded}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "agentainer_gpu.h"', 'int main(void) {']
    for cname, ct in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    for cname, dt in (("agr_record", A.record_dtype), ("agr_outcome", A.outcome_dtype), ("agr_verdict", A.verdict_dtype),
                      ("agr_dispatch", A.dispatch_dtype)):
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname in dt.names:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for cname, ct in structs.items():
        assert int(got[cname]) == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(ct, fname).offset, f"{cname}.{fname}"
    for cname, dt in (("agr_record", A.record_dtype), ("agr_outcome", A.outcome_dtype), ("agr_verdict", A.verdict_dtype),
                      ("agr_dispatch", A.dispatch_dtype)):
        assert int(got[cname]) == dt.itemsize, cname
        for fname in dt.names:
            assert int(got[f"{cname}.{fname}"]) == dt.fields[fname][1], f"{cname}.{fname}"


def test_integration_text_only_names_what_the_header_declares():
    """The cgo shim in INTEGRATION.md cannot be compiled here (no Go toolchain); at least every C function, constant and
    struct field it names must exist in the header it binds."""
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    syms = set(declared_symbols())
    used = set(re.findall(r"\bC\.(agr_[a-z0-9_]+)\(", text))
    assert used and used <= syms, sorted(used - syms)
    body = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    for name in set(re.findall(r"\bC\.(AGR_[A-Z0-9_]+)\b", text)):
        assert re.search(rf"\b{name}\b", body), name
    for st in set(re.findall(r"\bC\.(agr_[a-z_]+)\{", text)) | set(re.findall(r"var \w+ C\.(agr_[a-z_]+)\b", text)):
        assert re.search(rf"typedef (struct {st}\b|\w+ {st};)", body), st
