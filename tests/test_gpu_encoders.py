"""og_encode_pages against the oracle's restated encoders, byte for byte, on the inputs where the codec choice turns.

The expected page is oracle.field_page_encode / oracle.time_page_encode, except where the reference hands the block to a
third-party codec (encode.cu, DESIGN.md "Deviations"): there the device writes the uncompressed form of the same block, restated
here from the Go sources:
  floats, Snappy (few decimals, NaN) or a Gorilla refusal   compact_model.raw_float_page   [hdr][0x00][values LE]
  ints, zstd (a zig-zag delta above 2^60 - 1)               int.go uncompressedData        [hdr][0x40][u32 BE 8n][zig-zag BE ...]
  times, Snappy (a delta of 2^60 - 1 or more)               timestamp.go packUncompressedData  [32][u32 BE n][0x40][u32 BE 8n][zig-zag BE ...]
A float segment with +Inf and -Inf (FloatArrayEncodeAll refuses it) makes og_encode_pages return OG_E_INVAL.

Every case is also run as one segment of a multi-segment call, cells at an rps stride, so the kernel's addressing of cells,
validity bytes and the dense-int scratch is pinned at the same time."""
import ctypes as C
import struct

import numpy as np
import pytest

import compact_model as cm
import oracle
import page_forms as pf
from opengemini_b200 import Shard
from opengemini_b200 import _lib as L

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = pf.I64_MIN, pf.I64_MAX
S8B_MAX = (1 << 60) - 1
PAGE_STRIDE = 8704
TIME = pf.TIME


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------- the call and the expected pages
def device_pages(typ, segs, rps=1000):
    """segs: [(cells per row, valid per row or None)] of one type (TIME: times, valid None) -> og_encode_pages' pages, one call,
    segment g's cells at rows [g * rps, g * rps + rows).  Returns the pages, or the status when the call refuses."""
    import torch
    n = len(segs)
    is_time = typ == TIME
    dt = np.uint8 if typ == L.TYPE_BOOL else np.int64 if typ in (TIME, L.TYPE_INT) else np.float64
    cells = np.zeros(n * rps, dt)
    ok = np.zeros(n * rps, np.uint8)
    rows = np.array([np.asarray(c).size for c, _v in segs], np.int32)
    with_valid = any(v is not None for _c, v in segs)
    for g, (c, v) in enumerate(segs):
        c = np.asarray(c, dt)
        assert 1 <= c.size <= rps
        cells[g * rps:g * rps + c.size] = c
        ok[g * rps:g * rps + c.size] = 1 if v is None else np.asarray(v, np.uint8)
        # rows past a segment's end hold garbage an encoder must not read
        cells[g * rps + c.size:(g + 1) * rps] = np.frombuffer(np.full((rps - c.size) * cells.itemsize, 0xA5, np.uint8), dt)
        ok[g * rps + c.size:(g + 1) * rps] = 1
    d_cells = torch.from_numpy(cells.view(np.uint8)).cuda()
    d_ok = torch.from_numpy(ok).cuda()
    d_rows = torch.from_numpy(rows).cuda()
    cap = n * PAGE_STRIDE
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    off = torch.zeros(n, dtype=torch.int64, device="cuda")
    ln = torch.zeros(n, dtype=torch.int32, device="cuda")
    total = C.c_uint64()
    st = L.lib().og_encode_pages(L.TYPE_INT if is_time else typ, 1 if is_time else 0, d_cells.data_ptr(),
                                 d_ok.data_ptr() if with_valid and not is_time else None, d_rows.data_ptr(), n, rps,
                                 out.data_ptr(), cap, off.data_ptr(), ln.data_ptr(), C.byref(total))
    if st != L.OG_OK:
        return st
    blob, offs, lens = out.cpu().numpy(), off.cpu().numpy(), ln.cpu().numpy().astype(np.int64)
    assert int(total.value) == int(lens.sum())
    assert np.array_equal(offs, np.concatenate([[0], np.cumsum(lens)[:-1]]))  # back to back, in segment order
    return [blob[int(o):int(o) + int(k)] for o, k in zip(offs, lens)]


def raw_time_page(t):
    t = np.asarray(t, np.int64)
    return np.frombuffer(struct.pack(">BIBI", 32, t.size, 0x40, 8 * t.size) + cm.zigzag_be(t), np.uint8)


def want_page(typ, cells, valid=None):
    """the page og_encode_pages must write; None where it must refuse the segment (+Inf and -Inf)"""
    if typ == TIME:
        p = oracle.time_page_encode(np.asarray(cells, np.int64))
        return raw_time_page(cells) if pf.time_codec(p) == "t_snappy" else p
    valid = np.ones(np.asarray(cells).size, bool) if valid is None else np.asarray(valid, bool)
    try:
        p = oracle.field_page_encode(typ, np.ascontiguousarray(cells), None if valid.all() else valid.astype(np.uint8))
    except ValueError:
        if typ == L.TYPE_FLOAT:
            return None
        assert typ == L.TYPE_INT
        return cm.raw_int_page(cells, valid)
    if typ == L.TYPE_FLOAT and pf.codec_of(typ, p) == "snappy":
        return cm.raw_float_page(np.asarray(cells, np.float64), valid)
    return p


def check(typ, cases, rps=1000, labels=None):
    """cases: [(cells, valid or None)]: each alone and all in one call"""
    want = [want_page(typ, c, v) for c, v in cases]
    labels = labels or [str(i) for i in range(len(cases))]
    for (c, v), w, lab in zip(cases, want, labels):
        got = device_pages(typ, [(c, v)], rps)
        if w is None:
            assert got == L.OG_E_INVAL, lab
            continue
        assert not isinstance(got, int), (lab, got)
        assert np.array_equal(got[0], w), f"{lab}: device {got[0].size} B {bytes(got[0][:24]).hex()}, want {w.size} B {bytes(w[:24]).hex()}"
    keep = [k for k, w in enumerate(want) if w is not None]
    if len(keep) > 1:
        got = device_pages(typ, [cases[k] for k in keep], rps)
        for k, g in zip(keep, got):
            assert np.array_equal(g, want[k]), f"{labels[k]} in a call of {len(keep)} segments"
    return want


def _zz(d):
    """zig-zag encodings -> the int64 deltas that have them"""
    return [(z >> 1) ^ -(z & 1) for z in d]


def _walk(first, deltas):
    """int64 values first, first + d0, ... with wrapping sums"""
    v = np.cumsum(np.array([int(first)] + [int(x) for x in deltas], dtype=object))
    return np.array([int(x) & ((1 << 64) - 1) for x in v], np.uint64).view(np.int64)


# ---------------------------------------------------------------- time pages
def test_time_catalogue():
    es = pf.time_entries()
    want = check(TIME, [(e.cells, None) for e in es], labels=[e.name for e in es])
    for e, w in zip(es, want):
        assert np.array_equal(w, e.page), e.name


def _time_cases():
    rng = np.random.default_rng(7)
    T0, SEC = pf.T0, pf.SEC
    out = {"n1": [T0], "n2": [T0, T0 + 3], "n3": [T0, T0 + 3, T0 + 5], "n3_const": [T0, T0 + 4, T0 + 8],
           "const": T0 + np.arange(1000, dtype=np.int64) * 7}
    # multiples of 10, the last one not of 100: the search from the last delta never tries 10, so scale 1; when the last delta
    # is a multiple of 100, the step-down over the earlier deltas does reach 10
    d = np.concatenate([rng.integers(1, 40, 998) * 10, [30]])
    out["tens"] = T0 + np.concatenate([[0], np.cumsum(d)])
    out["tens_last_100"] = T0 + np.concatenate([[0], np.cumsum(np.concatenate([d[:-1], [1000]]))])
    # the scale steps down as earlier deltas are read: the last delta is 10^12, the ones before it 10^9, 10^6, 10^3 (then 1)
    d = np.concatenate([rng.integers(1, 9, 50) * 1000, rng.integers(1, 9, 50) * 10**6, rng.integers(1, 9, 50) * 10**9, [10**12]])
    out["scale_steps"] = T0 + np.concatenate([[0], np.cumsum(d)])
    out["scale_steps_to_1"] = T0 + np.concatenate([[0], np.cumsum(np.concatenate([[7], d]))])
    for k in range(1, 13):  # every scale the search can settle on
        out[f"scale_1e{k}"] = -(10**17) + np.concatenate([[0], np.cumsum(rng.integers(1, 30, 200) * 10**k)]).astype(np.int64)
    # one delta of 2^60 - 2 (Simple8b, a 60-bit value) and one of 2^60 - 1 (raw)
    base = -(1 << 62)
    out["delta_s8b_max"] = np.array([base, base + 1000, base + 1000 + S8B_MAX - 1, base + 2000 + S8B_MAX - 1], np.int64)
    out["delta_raw"] = np.array([base, base + 1000, base + 1000 + S8B_MAX, base + 2000 + S8B_MAX], np.int64)
    out["delta_raw_first"] = np.array([base, base + S8B_MAX, base + S8B_MAX + 5, base + S8B_MAX + 7], np.int64)
    out["delta_raw_long"] = np.concatenate([[base], base + S8B_MAX + np.cumsum(rng.integers(1, 1 << 40, 999))]).astype(np.int64)
    out["negative"] = -5 * 10**17 + np.cumsum(rng.integers(1, 10**6, 1000)).astype(np.int64)
    out["cross0"] = -500 + np.cumsum(rng.integers(1, 3, 1000)).astype(np.int64)
    out["near_min"] = I64_MIN + np.cumsum(rng.integers(0, 5, 1000) + 1).astype(np.int64) - 1
    out["near_min_const"] = I64_MIN + np.arange(1000, dtype=np.int64) * 3
    out["near_max"] = (I64_MAX - np.cumsum(rng.integers(1, 6, 1000))[::-1] + 1).astype(np.int64)
    out["near_max_const"] = I64_MAX - 999 * 5 + np.arange(1000, dtype=np.int64) * 5
    out["min_to_max"] = np.array([I64_MIN, I64_MIN + 1, 0, I64_MAX - 1, I64_MAX], np.int64)
    out["min_max2"] = np.array([I64_MIN, I64_MAX], np.int64)
    return {k: np.asarray(v, np.int64) for k, v in out.items()}


def test_time_edges():
    cases = _time_cases()
    want = check(TIME, [(t, None) for t in cases.values()], labels=list(cases))
    got = dict(zip(cases, want))
    # the forms the cases exist for
    assert pf.time_codec(got["n1"]) == "t_one" and pf.time_codec(got["n2"]) == "t_raw" and pf.time_codec(got["n3_const"]) == "t_const"
    assert pf.time_s8b(got["tens"])[0] == 1 and pf.time_s8b(got["tens_last_100"])[0] == 10
    assert pf.time_s8b(got["scale_steps"])[0] == 1000 and pf.time_s8b(got["scale_steps_to_1"])[0] == 1
    for k in range(2, 13):
        assert pf.time_s8b(got[f"scale_1e{k}"])[0] == 10**k, k
    assert pf.time_s8b(got["scale_1e1"])[0] == 1
    assert pf.time_codec(got["delta_s8b_max"]) == "t_s8b" and 15 in pf.time_s8b(got["delta_s8b_max"])[1]
    for k in ("delta_raw", "delta_raw_first", "delta_raw_long", "min_to_max"):
        assert pf.time_codec(got[k]) == "t_raw", k
    assert pf.time_codec(got["near_min_const"]) == pf.time_codec(got["near_max_const"]) == "t_const"
    for k, t in cases.items():  # and every page decodes to its times
        assert np.array_equal(oracle.time_page_decode(got[k]), t), k


# ---------------------------------------------------------------- int pages
ONES = {119: set(), 120: {1}, 239: {1}, 240: {0}, 241: {0}, 360: {0, 1}}  # the selectors 0 / 1 the run of ones takes


def _int_cases():
    rng = np.random.default_rng(11)
    out = {}
    out["const_wrap"] = _walk(I64_MAX - 10, [3] * 999)                       # the sums wrap past INT64_MAX
    out["const_wrap_neg"] = _walk(I64_MIN + 10, [-7] * 500)
    out["const_huge_delta"] = _walk(I64_MIN, [I64_MAX] * 3)                   # zig-zag delta 2^64 - 2: const, not Simple8b
    out["zz_s8b_max"] = _walk(5, _zz([S8B_MAX, 3, 1, 8]))                      # zig-zag 2^60 - 1: Simple8b
    out["zz_raw"] = _walk(5, _zz([1 << 60, 3, 1, 8]))                          # zig-zag 2^60: raw
    out["zz_raw_last"] = _walk(5, _zz(list(rng.integers(0, 1 << 20, 500)) + [1 << 60]))
    out["zz_s8b_max_long"] = _walk(-3, _zz(list(rng.integers(0, 1 << 20, 500)) + [S8B_MAX]))
    for k in ONES:  # canPack takes 240 / 120 ones only as the rest; 30 twos fill one word, so the run starts a word
        out[f"ones{k}"] = _walk(3, _zz([2] * 30 + [1] * k))
        out[f"ones{k}_then"] = _walk(3, _zz([2] * 30 + [1] * k + [6]))
    out["minmax"] = np.array([I64_MIN, I64_MAX, I64_MIN, 0, I64_MAX, -1], np.int64)
    out["min_step"] = I64_MIN + np.cumsum(rng.integers(0, 3, 1000)).astype(np.int64)
    out["max_step"] = I64_MAX - np.cumsum(rng.integers(0, 3, 1000))[::-1].astype(np.int64)
    out["random_full"] = rng.integers(I64_MIN, I64_MAX, 1000, dtype=np.int64, endpoint=True)
    out["n1_min"] = np.array([I64_MIN], np.int64)
    out["n2"] = np.array([I64_MAX, 4], np.int64)
    out["n3"] = np.array([1, 2, 4], np.int64)
    cases = {k: (v, None) for k, v in out.items()}
    # nulls at 0 / 5 / 40 / 99 / 100 %, under every codec (the dense-int scratch path): walks, constants, raw
    for null_p in (0.0, 0.05, 0.4, 0.99, 1.0):
        for kind in ("walk", "const", "raw", "s8b_edge"):
            n = int(rng.integers(900, 1001))
            if kind == "walk":
                v = rng.integers(-50, 50, n).cumsum()
            elif kind == "const":
                v = 17 + 5 * np.arange(n, dtype=np.int64)
            elif kind == "raw":
                v = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64)
            else:
                v = np.asarray(_walk(0, _zz([S8B_MAX, S8B_MAX - 1] * (n // 2))[:n - 1]))
            ok = rng.random(n) >= null_p
            if null_p in (0.05, 0.4):
                ok[0] = ok[-1] = False
            v = np.where(ok, v, 0).astype(np.int64)
            v[~ok] = rng.integers(-9, 9, int((~ok).sum()))  # cells under nulls hold garbage
            cases[f"nulls{null_p}_{kind}"] = (v, ok)
    return cases


def test_int_edges():
    cases = _int_cases()
    want = dict(zip(cases, check(L.TYPE_INT, list(cases.values()), labels=list(cases))))
    codec = {k: pf.codec_of(L.TYPE_INT, w) for k, w in want.items()}
    assert codec["const_wrap"] == codec["const_huge_delta"] == "const"
    assert codec["zz_s8b_max"] == codec["zz_s8b_max_long"] == "s8b" and codec["zz_raw"] == codec["zz_raw_last"] == "raw"
    assert codec["minmax"] == codec["nulls0.4_raw"] == "raw" and codec["nulls0.0_s8b_edge"] == "s8b" and codec["nulls0.0_const"] == "const"

    def sels(k):
        return set(pf.s8b_selectors(pf.int_block_words(pf.read_header(want[k])["block"]))) & {0, 1}
    for k, s01 in ONES.items():  # a non-1 value after the run: canPack's "all remaining" is false, no selector 0 / 1
        assert sels(f"ones{k}") == s01 and sels(f"ones{k}_then") == set(), k


# ---------------------------------------------------------------- float pages
def _gorilla_limit_cases():
    """segments whose Gorilla block is exactly at the 90 %-of-raw limit (kept) and one byte over it (raw): random doubles (no
    few-decimal shortcut) for the first k values, then the last one repeated; k and the row count searched on the oracle"""
    rng = np.random.default_rng(5)
    dense = rng.standard_normal(1000) * 1e3
    at, over = {}, {}
    for n in range(1000, 400, -1):
        limit = n * 8 * 90 // 100
        lo, hi = 10, n
        size = lambda k: oracle._enc("ogo_gorilla_encode", np.concatenate([dense[:k], np.full(n - k, dense[k - 1])]), 16 * n + 64).size + 1
        while hi - lo > 1:  # the largest k whose block fits
            m = (lo + hi) // 2
            lo, hi = (m, hi) if size(m) <= limit else (lo, m)
        for k in (lo, lo + 1):
            s = size(k)
            v = np.concatenate([dense[:k], np.full(n - k, dense[k - 1])])
            if s == limit and "at" not in at:
                at["at"] = v
            if s == limit + 1 and "over" not in over:
                over["over"] = v
        if at and over:
            break
    assert at and over
    return {"gorilla_at_limit": at["at"], "gorilla_over_limit": over["over"]}


def _float_cases():
    rng = np.random.default_rng(13)
    r = lambda n: rng.integers(-(1 << 20), 1 << 20, n) / 1024.0 + 0.5 ** 11  # noqa: E731  (short mantissas, not few decimals)
    out = {"n4": r(4), "n5": r(5), "n4_nan": np.array([1.5, np.nan, 2.0, 3.0]), "n1": r(1), "n2_infs": np.array([np.inf, -np.inf])}
    for nd in (1, 8, 9):
        vals = r(nd)
        out[f"distinct{nd}"] = np.repeat(vals, 1000 // nd + 1)[:1000]
        # -0.0 first, then nd - 1 other values (nd = 1: zeros): the reference compares floats, so -0.0 is stored as a zero
        rest = np.repeat(vals[1:], 999 // max(1, nd - 1) + 1)[:999] if nd > 1 else np.zeros(999)
        out[f"distinct{nd}_negzero_first"] = np.concatenate([[-0.0], rest])
    out["same_negzero"] = np.full(1000, -0.0)
    out["same_negzero_then_zero"] = np.array([-0.0] * 3 + [0.0] * 500)
    out["same_zero_then_negzero"] = np.array([0.0] * 3 + [-0.0] * 500)
    out["rle_signed_zeros"] = np.repeat([0.0, -0.0, 1.0, -0.0, 0.0, 2.5], [100, 50, 10, 300, 7, 33])
    out["rle_all_zeros_mix"] = np.tile([0.0, -0.0], 400)
    out.update(_gorilla_limit_cases())
    out["few_decimal"] = np.round(r(1000), 2)
    out["few_decimal_int"] = np.round(r(1000))                       # integers: Gorilla
    out["nan"] = np.where(rng.random(1000) < 0.1, np.nan, r(1000))
    out["nan_first"] = np.concatenate([[np.nan], r(999)])
    out["inf_pos"] = np.where(rng.random(1000) < 0.02, np.inf, r(1000))
    out["inf_neg"] = np.where(rng.random(1000) < 0.02, -np.inf, r(1000))
    out["inf_both"] = np.concatenate([r(1), [np.inf], r(500), [-np.inf], r(497)])  # refused
    out["inf_both_first"] = np.concatenate([[-np.inf], [np.inf], r(998)])          # the running sum skips the first value: kept
    cases = {k: (np.asarray(v, np.float64), None) for k, v in out.items()}
    for null_p in (0.05, 0.4, 0.99):
        n = 1000
        ok = rng.random(n) >= null_p
        if null_p < 0.5:
            ok[0] = ok[-1] = False
        for kind, v in (("gorilla", r(n)), ("rle", np.repeat(r(4), 250)), ("same_negzero", np.full(n, -0.0)), ("few_dec", np.round(r(n), 1))):
            cases[f"nulls{null_p}_{kind}"] = (np.where(ok, v, rng.random(n)), ok)
    return cases


def test_float_edges():
    cases = _float_cases()
    want = dict(zip(cases, check(L.TYPE_FLOAT, list(cases.values()), labels=list(cases))))
    codec = {k: pf.codec_of(L.TYPE_FLOAT, w) for k, w in want.items() if w is not None}
    assert want["inf_both"] is None and want["n2_infs"] is not None and codec["inf_both_first"] == "gorilla"
    assert codec["n4"] == codec["n4_nan"] == "raw" and codec["n5"] == "rle"
    assert codec["distinct1"] == codec["distinct1_negzero_first"] == "same" and codec["distinct8"] == codec["distinct8_negzero_first"] == "rle"
    assert codec["distinct9"] == codec["distinct9_negzero_first"] == "gorilla"
    assert want["distinct1_negzero_first"].size == 5 + 1 + 2  # Same of zeros: no value stored, -0.0 included
    assert codec["gorilla_at_limit"] == "gorilla" and codec["gorilla_over_limit"] == "raw"
    assert codec["few_decimal"] == codec["nan"] == codec["nan_first"] == "raw" and codec["few_decimal_int"] == "gorilla"
    assert codec["inf_pos"] == codec["inf_neg"] == "gorilla"


# ---------------------------------------------------------------- bool pages
def test_bool_null_bitmap_edges():
    rng = np.random.default_rng(17)
    cases, labels = [], []
    for n in (1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 257, 999, 1000):
        v = (rng.random(n) < 0.5).astype(np.uint8)
        for where in ("none", "first", "last", "byte_edges", "all", "all_but_one", "random"):
            ok = np.ones(n, bool)
            if where == "first":
                ok[0] = False
            elif where == "last":
                ok[-1] = False
            elif where == "byte_edges":
                ok[[i for i in range(n) if i % 8 in (0, 7)]] = False
            elif where == "all":
                ok[:] = False
            elif where == "all_but_one":
                ok[:] = False; ok[n // 2] = True
            elif where == "random":
                ok = rng.random(n) >= 0.3
            cases.append((np.where(ok, v, rng.integers(2, 255, n)).astype(np.uint8), None if where == "none" else ok))
            labels.append(f"{n} {where}")
    check(L.TYPE_BOOL, cases, labels=labels)


# ---------------------------------------------------------------- many segments per call
def _random_segment(typ, rng, n):
    """one segment of n rows from a mix of generators (codecs, nulls, specials)"""
    kind = int(rng.integers(0, 6))
    null_p = [0.0, 0.0, 0.05, 0.4, 0.99, 1.0][int(rng.integers(0, 6))]
    ok = rng.random(n) >= null_p
    if typ == TIME:
        step = [1, 10, 1000, 10**9, 7, 1 << 59][kind]
        d = rng.integers(1, 4, n - 1) * step if kind != 2 else np.full(n - 1, step)
        return np.concatenate([[int(rng.integers(-(1 << 61), 1 << 61))], d]).cumsum().astype(np.int64), None
    if typ == L.TYPE_BOOL:
        v = (rng.random(n) < [0.5, 0.0, 1.0, 0.9, 0.1, 0.5][kind]).astype(np.uint8)
    elif typ == L.TYPE_INT:
        v = [lambda: rng.integers(-100, 100, n).cumsum(), lambda: np.full(n, int(rng.integers(-5, 5))) + np.arange(n) * 3,
             lambda: rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64), lambda: rng.integers(0, 2, n).cumsum(),
             lambda: (I64_MAX - rng.integers(0, 1 << 20, n)), lambda: np.asarray(_walk(0, _zz(rng.integers(S8B_MAX - 1, S8B_MAX + 2, n - 1).tolist())))][kind]()
    else:
        v = [lambda: rng.standard_normal(n) * 100, lambda: np.repeat(rng.standard_normal(3), n // 3 + 1)[:n],
             lambda: np.full(n, [0.0, -0.0, 2.5][int(rng.integers(0, 3))]), lambda: np.round(rng.standard_normal(n) * 100, 2),
             lambda: np.where(rng.random(n) < 0.05, np.nan, rng.standard_normal(n)),
             lambda: np.where(rng.random(n) < 0.05, np.inf, rng.integers(-50, 50, n).astype(np.float64))][kind]()
    v = np.asarray(v)
    return v, (None if ok.all() and rng.random() < 0.5 else ok)


@pytest.mark.parametrize("rps", [1, 7, 999, 1000])
@pytest.mark.parametrize("typ", [L.TYPE_FLOAT, L.TYPE_INT, L.TYPE_BOOL, TIME], ids=["float", "int", "bool", "time"])
def test_many_segments_in_one_call(typ, rps):
    """about 2000 segments (fewer for long ones) of 1..rps rows in one call; each page compared at its page_off / page_len"""
    rng = np.random.default_rng(rps * 10 + typ)
    n_seg = 2000 if rps < 999 else 600
    segs = [_random_segment(typ, rng, int(rng.integers(1, rps + 1))) for _ in range(n_seg)]
    if typ != TIME and not any(v is not None for _c, v in segs):
        segs[0] = (segs[0][0], np.ones(segs[0][0].size, bool))
    want = [want_page(typ, c, v) for c, v in segs]
    assert all(w is not None for w in want)
    got = device_pages(typ, segs, rps)
    assert not isinstance(got, int), got
    for g, (w, gg) in enumerate(zip(want, got)):
        assert np.array_equal(gg, w), f"segment {g} of {n_seg} ({segs[g][0].size} rows): device {gg.size} B, want {w.size} B"


def test_refusal_of_one_segment_fails_the_call():
    """+Inf and -Inf in one segment among others: the whole call is refused"""
    rng = np.random.default_rng(19)
    segs = [(rng.standard_normal(50), None) for _ in range(30)]
    segs[17] = (np.concatenate([rng.standard_normal(1), [np.inf], rng.standard_normal(47), [-np.inf]]), None)
    assert device_pages(L.TYPE_FLOAT, segs, 50) == L.OG_E_INVAL
    assert "FloatArrayEncodeAll" in L.lib().og_last_error().decode()
