"""CPU tests (no GPU) of embedding dropout (fit(entity_dropout=..., relation_dropout=...); DESIGN.md 3.19): fit's
refusals, each before anything is indexed; the oracle's mask stream against plain Python on oracle/philox.py, with
pinned words; the kept fraction; the workspace formulas; the header and the ctypes table."""
import ctypes as C
import math
import re

import numpy as np
import pytest

import dropout_oracle as do
from ampligraph_b200 import _lib
from ampligraph_b200.engine import (dropout_workspace_bytes, k_vs_all_workspace_bytes, one_vs_all_relation_workspace_bytes,
                                    one_vs_all_workspace_bytes)
from oracle import philox

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


def _model(scoring="ComplEx", loss="multiclass_nll"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)
    m.compile(optimizer="adam", loss=loss)
    return m


@pytest.mark.parametrize("which", ["entity_dropout", "relation_dropout"])
@pytest.mark.parametrize("bad", [-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf"), "0.1", None, True, False,
                                 np.bool_(True), 1j])
def test_bad_values_refused_before_indexing(which, bad):
    m = _model()
    with pytest.raises(ValueError, match=which):
        m.fit(X, epochs=1, one_vs_all="s,o", **{which: bad})
    assert m.engine is None


@pytest.mark.parametrize("kw", [{}, {"focusE": True}])
def test_without_all_candidate_training_refused(kw):
    m = _model(loss="pairwise")
    with pytest.raises(ValueError, match="one_vs_all and k_vs_all"):
        m.fit(X, epochs=1, entity_dropout=0.3, **kw)
    assert m.engine is None
    with pytest.raises(ValueError, match="one_vs_all and k_vs_all"):
        m.fit(X, epochs=1, relation_dropout=0.3, **kw)
    assert m.engine is None


def test_with_user_loss_refused():
    m = _model(loss=lambda sp, sn: sp)
    with pytest.raises(ValueError, match="one_vs_all and k_vs_all"):
        m.fit(X, epochs=1, entity_dropout=0.3)
    assert m.engine is None


def test_with_focuse_and_one_vs_all_refused():
    m = _model()
    with pytest.raises(NotImplementedError, match="focusE"):
        m.fit(X, epochs=1, one_vs_all="o", entity_dropout=0.3, focusE=True)
    assert m.engine is None


def test_mask_words_restate_philox():
    """The numpy stream equals the plain-Python one on oracle/philox.py, counter by counter."""
    seed, step = 0x123456789ABCDEF0, 0x1_0000_0007
    for tg in (4, 9, 15):
        w = do.words(seed, step, tg, [0, 1, 77, 2 ** 31 - 1], 12)
        for i, row in enumerate([0, 1, 77, 2 ** 31 - 1]):
            for c in range(12):
                ctr = (row, (c >> 2) | ((0x80 | tg) << 24), step & 0xFFFFFFFF, step >> 32)
                want = philox.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[c & 3]
                assert int(w[i, c]) == want == do.mask_words(seed, step, tg, row, c)


def test_pinned_mask_words():
    """A few words of the stream, pinned: seed 0, step 0, tag 8 (side o's candidates), rows 0 and 1, columns 0 .. 4."""
    got = [do.mask_words(0, 0, 8, r, c) for r in (0, 1) for c in range(5)]
    assert got == PINNED, [hex(x) for x in got]


PINNED = [0x659328b3, 0x429aa419, 0xe0e88967, 0xd540a450, 0x3fea7089,
          0x11f59396, 0x9b139b52, 0xa75531d1, 0xba3c898c, 0xb75b2edf]


def test_tags_disjoint_from_the_other_streams():
    """Every dropout counter's word 1 has top byte 0x84 .. 0x8F; the corruption stream's is r >> 32 (0 below 2^56) and
    the negative samplers' the attempt index (< 0x80); the initialisers' c1 is a row index >> 32 or >> 34."""
    tags = [do.tag(s, r) for s in ("s", "o", "p") for r in range(4)]
    assert sorted(tags) == list(range(4, 16))
    assert all(0x84 <= (0x80 | t) <= 0x8F for t in tags)


@pytest.mark.parametrize("p", [0.1, 0.4, 0.5, 0.75])
def test_kept_fraction_within_five_sigma(p):
    n_rows, ld = 10 ** 6 // 100, 100
    k = do.keep(7, 3, do.tag("o", 0), np.arange(n_rows), ld, p)
    n = k.size
    assert n == 10 ** 6
    want = 1.0 - do.threshold(p) / 2.0 ** 24
    assert abs(want - (1.0 - p)) < 2.0 ** -24
    assert abs(k.mean() - want) <= 5 * math.sqrt(want * (1 - want) / n)


def test_threshold_and_scale():
    assert do.threshold(0.0) == 0 and do.threshold(0.5) == 2 ** 23 and do.threshold(0.75) == 3 * 2 ** 22
    assert do.scale(0.5) == np.float32(2.0) and do.scale(0.75) == np.float32(4.0)
    assert do.scale(0.4) == np.float32(1.0 / 0.6000000238418579)


def test_padded_columns():
    assert list(do.padded_columns("DistMult", 6)) == list(range(6))
    assert list(do.padded_columns("ComplEx", 12)) == [0, 1, 2, 3, 4, 5, 8, 9, 10, 11, 12, 13]


def test_workspace_formulas_add_two_candidate_tables():
    for B, n, ld in ((1, 2, 4), (1000, 14541, 200), (37, 300, 36)):
        extra = 2 * ((4 * n * ld + 15) // 16 * 16)
        assert dropout_workspace_bytes(n, ld, True) == extra and dropout_workspace_bytes(n, ld) == 0
        assert one_vs_all_workspace_bytes(B, n, ld, True) == one_vs_all_workspace_bytes(B, n, ld) + extra
        assert k_vs_all_workspace_bytes(B, n, ld, True) == k_vs_all_workspace_bytes(B, n, ld) + extra
        assert (one_vs_all_relation_workspace_bytes(B, n, ld, True)
                == one_vs_all_relation_workspace_bytes(B, n, ld) + extra)


def test_header_and_ctypes_table_agree():
    header = re.sub(r"/\*.*?\*/", "", open(_lib.HEADER).read(), flags=re.S)
    m = re.search(r"int\s+kge_set_embedding_dropout\s*\(([^)]*)\)", header)
    assert m, "kge_set_embedding_dropout is not declared"
    args = [a.strip() for a in m.group(1).split(",")]
    assert args == ["kge_handle *h", "float p_ent", "float p_rel", "uint64_t seed"]
    assert _lib.PROTOTYPES["kge_set_embedding_dropout"] == (C.c_int, [_lib._P, C.c_float, C.c_float, C.c_uint64])
