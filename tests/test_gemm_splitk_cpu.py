"""CPU-only checks of the skinny split-K plan's launch heuristics: the two tuning keys, their defaults and the
`ops.tuning` names that set them (the plan itself runs on the GPU: tests/test_gemm_splitk_gpu.py)."""
import os
import re

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tuning_keys_match_the_header_and_default_to_the_skinny_plan():
    from magicdance_b200 import _lib, ops
    with open(os.path.join(REPO, "include", "magicdance_b200.h")) as f:
        hdr = f.read()
    assert int(re.search(r"MDB_TUNE_GEMM_SKINNY_CTAS = (\d+)", hdr).group(1)) == _lib.TUNE_GEMM_SKINNY_CTAS
    assert int(re.search(r"MDB_TUNE_GEMM_SPLIT_MIN_CHUNKS = (\d+)", hdr).group(1)) == _lib.TUNE_GEMM_SPLIT_MIN_CHUNKS
    lib = _lib.load()
    assert lib.mdb_get_tuning(_lib.TUNE_GEMM_SKINNY_CTAS) == 96
    assert lib.mdb_get_tuning(_lib.TUNE_GEMM_SPLIT_MIN_CHUNKS) == 8
    with ops.tuning(skinny_ctas=0, split_min_chunks=16):
        assert lib.mdb_get_tuning(_lib.TUNE_GEMM_SKINNY_CTAS) == 0
        assert lib.mdb_get_tuning(_lib.TUNE_GEMM_SPLIT_MIN_CHUNKS) == 16
        assert lib.mdb_get_tuning(_lib.TUNE_GEMM_BN80_BELOW) == 100  # the other keys keep their own slots
        assert lib.mdb_get_tuning(_lib.TUNE_GEMM_PAIR_MIN_TILES) == 128
    assert lib.mdb_get_tuning(_lib.TUNE_GEMM_SKINNY_CTAS) == 96
    assert lib.mdb_get_tuning(_lib.TUNE_GEMM_SPLIT_MIN_CHUNKS) == 8


def test_unknown_tuning_key_is_refused():
    from magicdance_b200 import _lib
    lib = _lib.load()
    assert lib.mdb_set_tuning(7, 1) == -1
    assert "unknown key 7" in lib.mdb_last_error().decode()
    with pytest.raises(KeyError):
        from magicdance_b200 import ops
        ops.tuning(skinny=1)
