"""CPU checks for records longer than AGR_VAR_MAX_RECORD: the piece-wise checksum reference (tests/longref.py) against the
whole-record reference (tests/verifyref.py), and the max_record_bytes rules of agr_create, which are checked before any
device is looked for."""
import numpy as np
import pytest

import agentainer_lab_b200 as A
import longref as L
import verifyref as V
from agentainer_lab_b200 import constants as K

LENGTHS = [8208, 16384 - 16, 16384, 16384 + 16, 65536, 1 << 20, 1 << 26]


def _whole(blob, offs):
    n = len(offs) - 1
    return V.record_cksums(np.arange(n), blob, voff=offs[:-1].astype(np.int64), vlen=np.diff(offs.astype(np.int64)))


@pytest.mark.parametrize("length", LENGTHS)
def test_piece_sums_equal_whole_record_sums(length):
    rng = np.random.default_rng(length)
    lens = np.array([96, length, 112], dtype=np.int64)
    h = np.zeros(3, dtype=A.header_dtype)
    blob, offs = L.blob_from(h, lens, rng)
    assert (L.piece_cksums(blob, offs) == _whole(blob, offs)).all()


@pytest.mark.parametrize("residue", range(16))
def test_piece_boundary_at_every_residue_mod_16_words(residue):
    """cuts after 2048 + residue words (and records starting at every 16-byte residue mod 64 B) give the whole-record sums"""
    rng = np.random.default_rng(100 + residue)
    lens = np.array([96 + 16 * (residue % 4), 3 * 8192 + 16 * residue, 8192 + 16, 40000], dtype=np.int64)
    blob, offs = L.blob_from(np.zeros(4, dtype=A.header_dtype), lens, rng)
    whole = _whole(blob, offs)
    assert (L.piece_cksums(blob, offs, L.PIECE_WORDS + residue) == whole).all()
    assert (L.piece_cksums(blob, offs, 4 + residue) == whole).all()


def test_var_record_len_cap():
    h = np.zeros(1, dtype=A.header_dtype)
    h["path_len"], h["hdr_len"], h["body_len"] = 10, 20, 30000
    rec = h.view(np.uint8)
    assert A.var_record_len(rec) == K.AGR_VAR_MAX_RECORD
    assert A.var_record_len(rec, cap=1 << 20) == 96 + 30032 == L.stored_len(h, 1 << 20)[0]


def _create(**kw):
    try:
        A.Engine(slab_rows=256, max_agents=4, **kw).close()
        return 0, ""
    except A.AgrError as e:
        return e.code, str(e)


VAR = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN


@pytest.mark.parametrize("kw, rule", [
    (dict(flags=VAR, vslab_bytes=1 << 22, max_record_bytes=8200), "multiple of 16"),
    (dict(flags=VAR, vslab_bytes=1 << 22, max_record_bytes=4096), "multiple of 16 in [8192, 2^26]"),
    (dict(flags=VAR, vslab_bytes=1 << 28, max_record_bytes=(1 << 26) + 16), "multiple of 16 in [8192, 2^26]"),
    (dict(flags=VAR, vslab_bytes=1 << 20, max_record_bytes=(1 << 19) + 16), "vslab_bytes / 2"),
    (dict(flags=VAR, max_record_bytes=(1 << 17) + 16), "vslab_bytes / 2"),     # default vslab_bytes: 1024 * 256 rows
    (dict(flags=K.AGR_CFG_PERSISTENCE, max_record_bytes=1 << 16), "needs AGR_CFG_VARLEN"),
])
def test_bad_max_record_bytes_is_einval_before_any_device(kw, rule):
    code, msg = _create(**kw)
    assert code == K.AGR_EINVAL and rule in msg, msg


@pytest.mark.parametrize("kw", [
    dict(flags=VAR, max_record_bytes=0),
    dict(flags=VAR, max_record_bytes=8192),
    dict(flags=VAR, vslab_bytes=1 << 20, max_record_bytes=1 << 19),
    dict(flags=VAR, max_record_bytes=1 << 17, vslab_bytes=1 << 18),
    dict(flags=VAR, vslab_bytes=1 << 27, max_record_bytes=1 << 26),
])
def test_good_max_record_bytes_passes_the_rules(kw):
    """accepted values get as far as the device: AGR_ENODEV without one, an engine with one"""
    code, msg = _create(**kw)
    assert code in (0, K.AGR_ENODEV), msg


def test_config_field_sits_where_reserved_was():
    assert A.binding.AgrConfig.max_record_bytes.offset == 68 and A.binding.AgrConfig.max_record_bytes.size == 4
