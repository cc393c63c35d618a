"""The page-form catalogue (tests/page_forms.py) holds what it claims and decodes to what it was built from.

CPU only: the forms are read back with the catalogue's own walkers, the cells through the oracle's decoders, and every page the
restated Python encoder (golden/pyenc.py) can write must be byte-identical to the oracle's."""
import os
import sys

import numpy as np
import pytest

import oracle
import page_forms as pf
from opengemini_b200 import _lib as L

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import pyenc  # noqa: E402

VALUES = pf.value_entries()
TIMES = pf.time_entries()
ALL = VALUES + TIMES


def _decode(e):
    if e.typ == pf.TIME:
        return oracle.time_page_decode(e.page, cap=e.rows + 8), None
    return oracle.field_page_decode(e.typ, e.page, cap=e.rows + 8)


def _same_cells(e, vals, valid):
    assert np.array_equal(valid, e.valid), f"{e.name}: validity"
    want = e.cells[e.valid]
    if e.typ == L.TYPE_FLOAT:
        assert np.array_equal(vals.view(np.uint64), want.view(np.uint64)), f"{e.name}: values"
    else:
        assert np.array_equal(vals.astype(np.int64), want.astype(np.int64)), f"{e.name}: values"


@pytest.mark.parametrize("e", ALL, ids=[e.name for e in ALL])
def test_entry_holds_its_forms(e):
    assert not pf.check_forms(e)


def test_catalogue_covers_the_forms_the_kernels_branch_on():
    got = {e.name: pf.inspect(e) for e in ALL}
    assert max(g.get("run66", 0) for g in got.values()) >= 300
    g_leads = set().union(*(g.get("leads", set()) for g in got.values()))
    assert {0, 1, 2, 3} <= g_leads
    assert set(range(16)) <= set().union(*(g.get("selectors", set()) for n, g in got.items() if n.startswith("i_")))
    assert set(range(1, 8)) <= {g.get("bm_off", 0) for g in got.values()}
    codecs = {(e.typ, got[e.name]["codec"]) for e in ALL}
    for typ, names in ((L.TYPE_FLOAT, ["gorilla", "raw", "same", "rle", "one", "empty"]), (L.TYPE_INT, ["const", "s8b", "raw", "one", "empty"]),
                       (L.TYPE_BOOL, ["bits", "one", "empty"]), (pf.TIME, ["t_const", "t_s8b", "t_raw", "t_one"])):
        for c in names:
            assert (typ, c) in codecs, (typ, c)
    for e in VALUES:  # every codec with a bitmap too
        if got[e.name]["header"] == "full":
            assert any(n == e.name + "_nulls" and got[n]["header"] == "normal" for n in got), e.name


@pytest.mark.parametrize("e", ALL, ids=[e.name for e in ALL])
def test_entry_decodes_to_its_cells(e):
    vals, valid = _decode(e)
    if e.typ == pf.TIME:
        assert np.array_equal(vals, e.cells)
    else:
        _same_cells(e, vals, valid)


HAND = [e for e in ALL if not e.encoder_built and e.twin]


@pytest.mark.parametrize("e", HAND, ids=[e.name for e in HAND])
def test_hand_built_page_decodes_like_its_encoder_built_twin(e):
    assert e.note, f"{e.name}: a hand-built page says why"
    parts = [oracle.field_page_decode(e.typ, p, cap=e.rows + 8) for p in e.twin]
    vals = np.concatenate([v for v, _ in parts])
    valid = np.concatenate([k for _, k in parts])
    _same_cells(e, vals, valid)


ENC = [e for e in ALL if e.encoder_built]


@pytest.mark.parametrize("e", ENC, ids=[e.name for e in ENC])
def test_python_encoder_writes_the_same_bytes(e):
    if e.typ == pf.TIME:
        want = pyenc.time_page([int(x) for x in e.cells])
    else:
        conv = float if e.typ == L.TYPE_FLOAT else int
        want = pyenc.field_page(e.typ, [conv(x) for x in e.cells], [int(k) for k in e.valid])
    if want is None:
        pytest.skip("a codec pyenc does not restate (Snappy / zstd)")
    assert bytes(e.page) == want


def test_every_codec_has_a_bitmapped_page_that_path_5_and_the_device_encoder_take():
    """k_fused_cols takes segments of <= 1024 rows and og_encode_pages <= 1000, so each codec needs a page with a bitmap inside
    both bounds (hand-built raw pages aside: the encoders never write them), and every bm_off page must fit path 5"""
    got = {e.name: pf.inspect(e) for e in VALUES}
    full = {(e.typ, got[e.name]["codec"]) for e in VALUES if got[e.name]["header"] == "full"}
    small = {(e.typ, got[e.name]["codec"]) for e in VALUES if got[e.name]["header"] == "normal" and e.rows <= 1000 and e.encoder_built}
    assert full <= small, full - small
    assert all(e.rows <= 1000 for e in VALUES if got[e.name]["bm_off"])
