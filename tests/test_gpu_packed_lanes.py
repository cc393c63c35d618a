"""k_fused_il lanes stored as fixed-width XOR deltas ("packed") next to Gorilla lanes, against the oracle.

When the interleaved copy of a float column is built, every Full Gorilla or raw page is walked once: the OR of the XORs of
consecutive values gives the delta window [lead, lead + m).  A segment is stored as its first value and then m-bit deltas
when that takes fewer words than its Gorilla stream, and always when its page is raw.  _model() restates that rule and the
lane-group sizes in Python and is checked against og_stats.il_packed_segments and il_bytes on every shard here.

Every query runs under OG_Q_STRICT_ORDER (path 2, bitwise) and, where the data has no NaN, in the folded order (path 3: float
sums within test_gpu_parity's SUM_RTOL, and +0.0 / -0.0 compared as floats, DESIGN.md "Exactness")."""
import struct

import numpy as np
import pytest

import oracle
import page_forms as pf
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
from test_gpu_page_forms import _open, _zeros_unsigned
from test_gpu_parity import compare_dense

pytestmark = pytest.mark.gpu

T0, SEC = pf.T0, pf.SEC
N = 1000
ALL6 = ["count", "sum", "min", "max", "first", "last"]
PAD_WORDS, BATCH_ROWS, SUPER = 6, 16, 4096  # OG_IL_PAD_WORDS, OG_IL_B, OG_IL_SUPER


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------------------------------------------------------
# pages and values
# ---------------------------------------------------------------------------------------------------------------
def _raw_page(v):
    """Full raw page: [31][u32 rows][0x00][rows x 8 B LE]"""
    v = np.ascontiguousarray(v, np.float64)
    return np.concatenate([np.frombuffer(struct.pack(">BIB", 31, v.size, 0x00), np.uint8), v.view(np.uint8)])


def _gorilla_page(v):
    """Full Gorilla page: [31][u32 rows][0x30][0x10][8 B first][records], whatever the adaptive encoder would pick"""
    v = np.ascontiguousarray(v, np.float64)
    blk = oracle._enc("ogo_gorilla_encode", v, v.size * 10 + 64)
    assert blk[0] == 0x10
    return np.concatenate([np.frombuffer(struct.pack(">BIB", 31, v.size, 0x30), np.uint8), blk])


def _u2f(u):
    return np.asarray(u, np.uint64).view(np.float64)


def _values(kind, rng):
    """(values, page) of one segment of N rows"""
    if kind == "ghi":  # G-hi-like: [100, 101) on the 2^-46 grid, every delta inside bits 45..0
        return _gorilla_page(100 + rng.random(N))
    if kind == "walk":  # integer-valued walk that mostly stands still: '0' records keep Gorilla shorter
        return _gorilla_page(1000.0 + np.cumsum(rng.integers(-3, 4, N) * (rng.random(N) < 0.25)))
    if kind == "const":
        return _gorilla_page(np.full(N, 42.75))
    if kind == "raw_sign":  # random doubles with sign changes: a 64-bit window
        return _raw_page(rng.standard_normal(N) * 1e3)
    if kind == "pm0":  # +0.0 / -0.0 in turn: the window is bit 63 alone (lead 0, m 1)
        return _raw_page(np.where(np.arange(N) % 2 == 1, -0.0, 0.0))
    if kind == "sign_hi":  # the sign flips every row and bits 51..44 vary: window bits 63..44
        u = (np.arange(N, dtype=np.uint64) % np.uint64(2)) << np.uint64(63) | np.uint64(0x3FF8000000000000) | \
            rng.integers(0, 256, N, dtype=np.uint64) << np.uint64(44)
        return _gorilla_page(_u2f(u))
    if kind == "dense":  # 66-bit '10' records for 800 rows: 64-bit deltas would be longer
        return _gorilla_page(pf.lane_values("dense", rng, N))
    raise ValueError(kind)


# ---------------------------------------------------------------------------------------------------------------
# the choice rule and the group sizes
# ---------------------------------------------------------------------------------------------------------------
def _window(page):
    """(lead, m) of the XOR deltas of a page"""
    rows = struct.unpack(">I", page[1:5].tobytes())[0]
    v, _ = oracle.field_page_decode(L.TYPE_FLOAT, page, cap=rows + 8)
    u = v.view(np.uint64)
    acc = int(np.bitwise_or.reduce(u[1:] ^ u[:-1])) if u.size > 1 else 0
    if acc == 0:
        return 0, 0
    lead = 64 - acc.bit_length()
    trail = (acc & -acc).bit_length() - 1
    return lead, 64 - lead - trail


def _form(page):
    """('packed' | 'gorilla' | None, words incl. pad) of one value page (const-delta time pages only in this file)"""
    p = np.asarray(page, np.uint8)
    rows = struct.unpack(">I", p[1:5].tobytes())[0]
    if p[0] != 31 or rows < 2:
        return None, 0
    tag = int(p[5]) >> 4
    if tag == 3 and p[6] == 0x10:
        words, raw = (p.size - 7 + 3) // 4 + PAD_WORDS, False
    elif tag == 0 and p.size == 6 + 8 * rows:
        words, raw = 2 * rows + PAD_WORDS, True
    else:
        return None, 0
    _lead, m = _window(p)
    packed = 2 + ((rows - 1) * m + 31) // 32 + PAD_WORDS
    return ("packed", packed) if raw or packed < words else ("gorilla", words)


def _model(pages):
    """pages[series][segment] -> (packed segments, bytes of the interleaved copy): lane groups of 32 consecutive entries of one
    binning domain, sorted by (domain, words); a group's rows are its longest lane rounded up to the bulk-copy batch"""
    J = len(pages[0]) if all(len(s) == len(pages[0]) for s in pages) else 0
    ent = []
    for s, segs in enumerate(pages):
        for j, pg in enumerate(segs):
            form, words = _form(pg)
            if form:
                ent.append(((s // SUPER) * J + j if J else 0, words, form))
    ent.sort(key=lambda e: (e[0], e[1]))  # stable, like the device radix sort
    total = 0
    for d in sorted({e[0] for e in ent}):
        w = [e[1] for e in ent if e[0] == d]
        for g in range(0, len(w), 32):
            total += -(-max(w[g:g + 32]) // BATCH_ROWS) * BATCH_ROWS * 32 * 4
    return sum(e[2] == "packed" for e in ent), total


def _shard(kinds, seed, n_seg=2):
    rng = np.random.default_rng(seed)
    pages = [[_values(k, rng) for _ in range(n_seg)] for k in kinds]
    series = [[(T0 + (np.arange(N, dtype=np.int64) + g * N) * SEC, [pages[s][g]]) for g in range(n_seg)] for s in range(len(kinds))]
    sh, sd = _open(series, [L.TYPE_FLOAT])
    return sh, sd, pages, _model(pages)


def test_model_windows_and_choices():
    """the data of each kind has the window and takes the form its name promises (CPU side of the cases below)"""
    rng = np.random.default_rng(1)
    want = {"ghi": ("packed", (18, 46)), "walk": ("gorilla", None), "const": ("packed", (0, 0)), "raw_sign": ("packed", (0, 64)),
            "pm0": ("packed", (0, 1)), "sign_hi": ("packed", (0, 20)), "dense": ("gorilla", None)}
    for kind, (form, win) in want.items():
        page = _values(kind, rng)
        assert _form(page)[0] == form, kind
        if win:
            assert _window(page) == win, kind
    # G-hi-like: the window ends at bit 0; sign_hi's starts at bit 63
    lead, m = _window(_values("ghi", rng))
    assert 64 - lead - m == 0


# ---------------------------------------------------------------------------------------------------------------
# queries
# ---------------------------------------------------------------------------------------------------------------
def _canon_sum_nans(d, calls):
    """NaN sums as one bit pattern: x86 and the GPU produce different NaNs for Inf - Inf and NaN arithmetic"""
    for c, (f, _col) in zip(d["cols"], calls):
        if f == "sum":
            u = np.asarray(c["values"]).view(np.uint64).copy()
            u[np.isnan(u.view(np.float64))] = 0x7FF8000000000000
            c["values"] = u
    return d


def _run(sh, sd, model, calls, iv, tmin, tmax, label, folded=True, group="all", nan=False):
    """strict order (path 2) bitwise, then the folded order (path 3) for one-tagset queries; asserts the model's counts"""
    modes = [(L.Q_STRICT_ORDER, 2)] + ([(0, 3)] if folded and group == "all" else [])
    for flags, path in modes:
        q = AggQuery(sh, calls, iv, tmin, tmax, flags=flags, group=group).run()
        try:
            st = q.stats()
            assert st["path"] == path, f"{label}: path {st['path']}, wanted {path}"
            assert st["il_state"] == 1 and st["general_segments"] == 0, label
            assert (st["il_packed_segments"], st["il_bytes"]) == model, f"{label}: {st['il_packed_segments']}, {st['il_bytes']} != {model}"
            gpu = q.dense_host()
            ref = oracle.scan(sd, q.desc, threads=1)
        finally:
            q.close()
        if nan:
            gpu, ref = _canon_sum_nans(gpu, calls), _canon_sum_nans(ref, calls)
        if path == 3:
            gpu, ref = _zeros_unsigned(gpu), _zeros_unsigned(ref)
        compare_dense(gpu, ref, calls, len(calls) > 1, f"{label} [path {path}]", float_sum_exact=path != 3)


MIXED = ["ghi", "walk", "const", "raw_sign", "pm0", "sign_hi", "dense", "ghi"]


@pytest.fixture(scope="module")
def mixed():
    """48 series x 2 segments of every kind: each segment index is one binning domain of 48 lanes (a full and a partial group)"""
    sh, sd, pages, model = _shard([MIXED[s % len(MIXED)] for s in range(48)], seed=7)
    assert 0 < model[0] < 96
    yield sh, sd, model
    sh.close()


@pytest.mark.parametrize("iv", [60, 7])
def test_all_aggregates_with_their_times(mixed, iv):
    sh, sd, model = mixed
    tmax = T0 + (2 * N - 1) * SEC
    _run(sh, sd, model, [(f, 0) for f in ALL6], iv * SEC, T0, tmax, f"all six iv={iv}")
    for f in ALL6:
        _run(sh, sd, model, [(f, 0)], iv * SEC, T0, tmax, f"{f} iv={iv}")


def test_ranges_that_cut_segments_at_both_ends(mixed):
    sh, sd, model = mixed
    for lo, hi, iv in ((17 * SEC + 3, (2 * N - 5) * SEC, 60), (123 * SEC + 1, 777 * SEC, 7), (1001 * SEC, 1500 * SEC - 1, 45), (5 * SEC, 998 * SEC, 0)):
        _run(sh, sd, model, [("sum", 0), ("count", 0), ("max", 0), ("first", 0), ("last", 0), ("min", 0)], iv * SEC, T0 + lo, T0 + hi,
             f"range [{lo}, {hi}] iv={iv}")


def test_per_series_output(mixed):
    sh, sd, model = mixed
    _run(sh, sd, model, [(f, 0) for f in ALL6], 60 * SEC, T0 + 30 * SEC, T0 + (2 * N - 31) * SEC, "per series", group="series")


def test_multi_chunk_plan(mixed, monkeypatch):
    """32-series chunks: the partial lane group of each domain straddles no chunk, the full one runs in the first"""
    sh, sd, model = mixed
    monkeypatch.setenv("OGPU_CHUNK_SERIES", "32")
    _run(sh, sd, model, [("sum", 0), ("count", 0), ("max", 0), ("last", 0)], 60 * SEC, T0, T0 + (2 * N - 1) * SEC, "chunks of 32")
    _run(sh, sd, model, [("min", 0), ("first", 0)], 7 * SEC, T0 + 11 * SEC, T0 + (2 * N - 13) * SEC, "chunks of 32, cut range")


def test_lanes_that_drift_apart_beyond_the_ring():
    """one lane group per segment index: packed G-hi lanes (46 bits a row) and Gorilla lanes of 66-bit records, which run
    ~0.6 words a row ahead, so after ~100 rows the lanes are more than the 64-row ring apart"""
    kinds = ["ghi" if s % 2 else "dense" for s in range(24)]
    sh, sd, pages, model = _shard(kinds, seed=11)
    assert model[0] == 24  # the G-hi half, both segments
    tmax = T0 + (2 * N - 1) * SEC
    for calls in ([(f, 0) for f in ALL6], [("sum", 0), ("count", 0), ("max", 0)]):
        for iv in (60, 7):
            _run(sh, sd, model, calls, iv * SEC, T0, tmax, f"drift {calls} iv={iv}")
    _run(sh, sd, model, [("last", 0), ("min", 0)], 60 * SEC, T0, tmax, "drift per series", group="series")
    sh.close()


def test_nan_payloads_and_infinities_in_packed_lanes():
    """raw pages (always packed) holding NaNs with payloads, +Inf and -Inf; strict order only (DESIGN.md "Exactness")"""
    rng = np.random.default_rng(13)
    pages = []
    for s in range(6):
        v = rng.standard_normal(N) * 10
        u = v.view(np.uint64)
        u[rng.integers(0, N, 20)] = np.uint64(0x7FF0000000000001)  # signalling payload
        u[rng.integers(0, N, 20)] = np.uint64(0xFFF800000000BEEF)
        u[rng.integers(0, N, 20)] = np.uint64(0x7FF8000000000001)  # the Gorilla stream's end marker, as a value
        v[rng.integers(0, N, 10)] = np.inf
        v[rng.integers(0, N, 10)] = -np.inf
        if s == 0:
            v[0] = np.nan
        pages.append([_raw_page(v)])
    series = [[(T0 + np.arange(N, dtype=np.int64) * SEC, pg)] for pg in pages]
    sh, sd = _open(series, [L.TYPE_FLOAT])
    model = _model(pages)
    assert model[0] == 6
    for iv in (60, 7, 0):
        _run(sh, sd, model, [(f, 0) for f in ALL6], iv * SEC, T0, T0 + (N - 1) * SEC, f"nan iv={iv}", folded=False, nan=True)
        for f in ("min", "max", "first", "last"):
            _run(sh, sd, model, [(f, 0)], iv * SEC, T0 + 3 * SEC, T0 + (N - 4) * SEC, f"nan {f} iv={iv}", folded=False, nan=True)
    sh.close()


def test_raw_and_gorilla_pages_of_one_value_shape():
    """the same G-hi-like values as a raw and as a Gorilla page both become packed lanes; an integer walk stays Gorilla"""
    rng = np.random.default_rng(17)
    pages = []
    for s in range(40):
        v = 100 + rng.random(N)
        w = 1000.0 + np.cumsum(rng.integers(-3, 4, N) * (rng.random(N) < 0.25))
        pages.append([_raw_page(v) if s % 2 else _gorilla_page(v), _gorilla_page(w)])
    series = [[(T0 + (np.arange(N, dtype=np.int64) + g * N) * SEC, [pages[s][g]]) for g in range(2)] for s in range(40)]
    sh, sd = _open(series, [L.TYPE_FLOAT])
    model = _model(pages)
    assert model[0] == 40
    _run(sh, sd, model, [("sum", 0), ("count", 0), ("max", 0)], 60 * SEC, T0, T0 + (2 * N - 1) * SEC, "raw and gorilla")
    _run(sh, sd, model, [(f, 0) for f in ALL6], 7 * SEC, T0 + 9 * SEC, T0 + (2 * N - 9) * SEC, "raw and gorilla, cut")
    sh.close()
