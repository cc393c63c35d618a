"""A catalogue of column pages in the forms real openGemini files hold and synthetic shards never produce, with an inspector
that reads the forms back out of the page bytes.

Every entry names the forms it exists for (`Entry.forms`): Gorilla record kinds, stored leading counts, the longest run of long
records, Simple8b selectors, the bitmap offset.  `check_forms` reads them back with the walkers below, which restate the page
layout (SURVEY.md App. A) in plain Python and share no code with oracle/ or tests/golden/pyenc.py, so an encoder change that
quietly turns an entry into another codec fails the entry's CPU test instead of emptying the GPU tests of their purpose.

Pages come from the oracle's restated encoders (`oracle.field_page_encode` / `time_page_encode`) wherever the reference
writer would produce them.  The few forms it never writes are assembled by hand from the layout, and the builder says why;
such an entry carries `twin`, encoder-built pages that hold the same cells.

Layout reminders (big-endian unless noted):
  field page   Full [30+c][u32 rows][block] | Empty [40+c][u32 rows] | one row [16+c][LE value] |
               normal [type][u32 nb][bitmap nb B, LSB-first from bit bm_off][u32 bm_off][u32 nil][block]   (c: int 2, float 1, bool 3)
  float block  [tag<<4]: 0 raw (LE f64 each) | 3 Gorilla [0x10][u64 first][records] | 4 Same [u16 n][LE f64 unless 0.0] |
               5 RLE runs [u16 n, bit 15 = run of 0.0][LE f64 unless a zero run]
  int block    1 const-delta [u64 zz first][uvarint zz delta][uvarint n-1] | 2 Simple8b [u32 words+1][u32 n][u64 zz first][words] |
               4 raw [u32 8n][u64 zz each]
  bool block   [0x10][u32 n][bits, MSB first]
  time page    [32][u32 rows] + 1 const-delta [u64 t0][uvarint d][uvarint n-1] | 2 Simple8b [u64 scale][u32 words+1][u32 n][u64 t0][words] |
               4 raw [u32 8n][u64 zz each];  one row [18][LE i64]
"""
import struct
from dataclasses import dataclass, field

import numpy as np

import oracle
from opengemini_b200 import _lib as L

T0 = 1_700_000_000_000_000_000
SEC = 1_000_000_000
TIME = -1  # Entry.typ of a time page
DBL_MAX = np.finfo(np.float64).max
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
S8B_TABLE = [(240, 0), (120, 0), (60, 1), (30, 2), (20, 3), (15, 4), (12, 5), (10, 6), (8, 7), (7, 8), (6, 10), (5, 12), (4, 15),
             (3, 20), (2, 30), (1, 60)]


@dataclass
class Entry:
    name: str
    typ: int                 # L.TYPE_FLOAT / TYPE_INT / TYPE_BOOL, or TIME
    cells: np.ndarray        # one per row (float64 / int64 / uint8); 0 at null rows; the times for a time page
    valid: np.ndarray        # bool per row
    page: np.ndarray         # uint8
    forms: dict              # what check_forms must find in the page
    twin: list = None        # hand-built entries: encoder-built pages whose cells, concatenated, equal this entry's cells
    note: str = ""           # why a hand-built entry is hand-built
    encoder_built: bool = True
    tags: set = field(default_factory=set)

    @property
    def rows(self):
        return self.cells.size

    def times(self):
        return self.cells if self.typ == TIME else T0 + np.arange(self.rows, dtype=np.int64) * SEC


# ---------------------------------------------------------------------------------------------------------------
# inspector
# ---------------------------------------------------------------------------------------------------------------
def _u32(p, o):
    return struct.unpack(">I", bytes(p[o:o + 4]))[0]


def _u64(p, o):
    return struct.unpack(">Q", bytes(p[o:o + 8]))[0]


def _uvarint(p, o):
    x = s = 0
    while True:
        c = int(p[o]); o += 1
        x |= (c & 0x7F) << s; s += 7
        if c < 0x80:
            return x, o


def read_header(page):
    """dict(kind = full | empty | one | normal, rows (None for normal: the time page knows), nil, bm_off, bitmap, block)"""
    p = np.asarray(page, np.uint8)
    t = int(p[0])
    if 16 < t < 21:
        return dict(kind="one", rows=1, nil=1 if p.size == 1 else 0, bm_off=0, bitmap=None, block=p[1:])
    if 30 < t < 35:
        return dict(kind="full", rows=_u32(p, 1), nil=0, bm_off=0, bitmap=None, block=p[5:])
    if 40 < t < 45:
        return dict(kind="empty", rows=_u32(p, 1), nil=_u32(p, 1), bm_off=0, bitmap=None, block=p[5:5])
    nb = _u32(p, 1)
    return dict(kind="normal", rows=None, nil=_u32(p, 9 + nb), bm_off=_u32(p, 5 + nb), bitmap=p[5:5 + nb], block=p[13 + nb:])


FLOAT_CODECS = {0: "raw", 2: "snappy", 3: "gorilla", 4: "same", 5: "rle"}
INT_CODECS = {1: "const", 2: "s8b", 3: "zstd", 4: "raw"}


def codec_of(typ, page):
    h = read_header(page)
    if h["kind"] in ("one", "empty"):
        return h["kind"]
    tag = int(h["block"][0]) >> 4
    if typ == L.TYPE_FLOAT:
        return FLOAT_CODECS.get(tag, f"tag{tag}")
    if typ == L.TYPE_INT:
        return INT_CODECS.get(tag, f"tag{tag}")
    return "bits" if tag == 1 else f"tag{tag}"


class _BitReader:
    def __init__(self, data):
        self.s = "".join(f"{int(b):08b}" for b in data)
        self.p = 0

    def read(self, k):
        v = int(self.s[self.p:self.p + k], 2) if k else 0
        self.p += k
        return v


def gorilla_records(block, n):
    """The n-1 records after the first value of a Gorilla block (block[0] is the codec tag).  One dict per record:
    kind '0' | '10' | '11', bits (record length), lead (stored leading count of the window the record uses), m (meaningful
    bits, 64 for a stored 0), clz (true leading zeros of the XOR delta; None for '0')."""
    assert int(block[1]) == 0x10, "Gorilla stream header"
    r = _BitReader(block[10:])
    lead = m = None
    out = []
    for _ in range(n - 1):
        p0 = r.p
        if r.read(1) == 0:
            out.append(dict(kind="0", bits=1, lead=lead, m=0, clz=None))
            continue
        if r.read(1) == 0:
            kind = "10"
        else:
            kind = "11"
            lead = r.read(5)
            m = r.read(6) or 64
        v = r.read(m)
        assert v != 0, "a non-'0' record carries a non-zero delta"
        out.append(dict(kind=kind, bits=r.p - p0, lead=lead, m=m, clz=lead + m - v.bit_length()))
    return out


def s8b_selectors(words):
    return [int(w) >> 60 for w in words]


def int_block_words(block):
    """Simple8b words of an int block (tag 2)"""
    enc = _u32(block, 1)
    return [_u64(block, 17 + 8 * i) for i in range(enc - 1)]


def time_codec(page):
    p = np.asarray(page, np.uint8)
    if int(p[0]) == 18:
        return "t_one"
    tag = int(p[5]) >> 4
    return {1: "t_const", 2: "t_s8b", 3: "t_snappy", 4: "t_raw"}.get(tag, f"t_tag{tag}")


def time_s8b(page):
    """(scale, selectors) of a Simple8b time page"""
    p = np.asarray(page, np.uint8)
    scale, enc = _u64(p, 6), _u32(p, 14)
    return scale, s8b_selectors([_u64(p, 30 + 8 * i) for i in range(enc - 1)])


def rle_runs(block):
    """[(length, is_zero_run)] of an RLE float block"""
    out, o = [], 1
    while o + 2 <= block.size:
        n = struct.unpack(">H", bytes(block[o:o + 2]))[0]
        if n >> 15:
            out.append((n & 0x7FFF, True)); o += 2
        else:
            out.append((n, False)); o += 10
    return out


def longest_run(flags):
    best = cur = 0
    for f in flags:
        cur = cur + 1 if f else 0
        best = max(best, cur)
    return best


def inspect(e):
    """What the page holds, as far as the form claims go"""
    if e.typ == TIME:
        out = dict(codec=time_codec(e.page))
        if out["codec"] == "t_s8b":
            out["scale"], sels = time_s8b(e.page)
            out["selectors"] = set(sels)
        return out
    h = read_header(e.page)
    out = dict(header=h["kind"], bm_off=h["bm_off"], codec=codec_of(e.typ, e.page))
    nvals = int(e.valid.sum())
    if out["codec"] == "gorilla":
        recs = gorilla_records(h["block"], nvals)
        out["kinds"] = {k: sum(r["kind"] == k for r in recs) for k in ("0", "10", "11")}
        out["leads"] = {r["lead"] for r in recs if r["kind"] == "11"}
        out["window_leads"] = {r["lead"] for r in recs if r["kind"] != "0"}
        out["lead_pairs"] = {(r["lead"], r["clz"]) for r in recs if r["kind"] == "11"}
        out["m64"] = sum(r["kind"] == "11" and r["m"] == 64 for r in recs)
        out["run66"] = longest_run(r["bits"] >= 66 for r in recs)
        out["zero_frac"] = out["kinds"]["0"] / max(1, len(recs))
        # leading count 2 next to 0/1 inside one segment: windows of both sides of the k_fused_il fast-path edge
        out["lead_switches"] = sum(1 for a, b in zip(recs, recs[1:]) if a["lead"] is not None and b["lead"] is not None
                                   and (a["lead"] <= 1) != (b["lead"] <= 1))
    elif out["codec"] == "s8b":
        out["selectors"] = set(s8b_selectors(int_block_words(h["block"])))
    elif out["codec"] == "rle":
        runs = rle_runs(h["block"])
        out["rle_zero_runs"] = sum(z for _n, z in runs)
        out["rle_max_run"] = max(n for n, _z in runs)
    return out


def check_forms(e):
    """List of the claims in e.forms that the page does not meet"""
    got = inspect(e)
    bad = []
    for k, want in e.forms.items():
        if k in ("header", "codec", "bm_off", "scale"):
            ok = got.get(k) == want
        elif k in ("leads", "lead_pairs", "selectors"):
            ok = set(want) <= got.get(k, set())
        elif k == "leads_within":
            ok = got.get("window_leads", {None}) <= set(want)
        elif k.startswith("min_"):
            ok = got.get(k[4:], 0) >= want
        elif k.startswith("kinds_"):
            ok = got["kinds"][k[6:]] >= want
        else:
            raise KeyError(k)
        if not ok:
            bad.append(f"{e.name}: {k} wants {want}, page has {got.get(k, got.get('kinds'))}")
    return bad


# ---------------------------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------------------------
def _u2f(u):
    return np.asarray(u, np.uint64).view(np.float64)


def _fpage(v, valid=None):
    return oracle.field_page_encode(L.TYPE_FLOAT, np.asarray(v, np.float64), None if valid is None else np.asarray(valid, np.uint8))


def _full(typ, name, cells, forms, **kw):
    cells = np.asarray(cells)
    page = oracle.field_page_encode(typ, cells)
    return Entry(name, typ, cells, np.ones(cells.size, bool), page, forms, **kw)


def _pairs(v):
    """every value twice: half the records are '0', which keeps dense streams under the 90 %-of-raw threshold"""
    return np.repeat(np.asarray(v), 2)[:2 * (len(v))]


def lane_values(kind, rng, n=1000):
    """Float series for lane groups: 'dense' (a 64-bit window, then a 66-bit '10' record per row), 'zeros' (ten values in runs:
    '0' records), 'switch' (windows of leading count 2 and 0 in turn), 'lead2' (every delta at leading count 2)"""
    if kind == "dense":
        d = rng.standard_normal(n * 4 // 5) * np.where(rng.random(n * 4 // 5) < 0.5, -1.0, 1.0)
        d[1] = _u2f(d[:1].view(np.uint64) ^ np.uint64((1 << 63) | 1))[0]
        return np.concatenate([d, np.full(n - d.size, d[-1])])
    if kind == "switch":
        # 'switch': leading count 2 and leading count 0 switching inside one segment, in blocks of 50 rows.  A window of trailing count t
        # absorbs every later delta with as many leading and >= t trailing zeros, so: a leading-0 block keeps the low 40 bits of
        # the row before it (its windows have >= 40 trailing zeros), and a leading-2 block varies every bit (trailing ~0), so its
        # second row cannot reuse the leading-0 window; its first row only clears the sign and bit 62 (a reuse)
        u, prev = [], int(rng.integers(0, 1 << 61))
        for b in range(n // 50):
            for k in range(25):
                if b % 2 == 1:  # sign flips every row, bit 62 set, bits 40..60 random, low 40 bits kept
                    x = (1 << 62) | (int(rng.integers(0, 1 << 21)) << 40) | (prev & ((1 << 40) - 1)) | ((k % 2) << 63)
                elif k == 0:
                    x = prev & ((1 << 62) - 1)
                else:  # bit 61 differs from the row before: leading count exactly 2
                    x = int(rng.integers(0, 1 << 61)) | ((((prev >> 61) & 1) ^ 1) << 61)
                u.append(x); prev = x
        return _u2f(np.repeat(np.array(u, np.uint64), 2))
    if kind == "zeros":
        return np.repeat(rng.standard_normal(10) + 100, n // 10)
    u = rng.integers(0, 1 << 61, n // 2, dtype=np.uint64) | (np.arange(n // 2, dtype=np.uint64) % np.uint64(2)) << np.uint64(61)
    return _u2f(np.repeat(u, 2))


def float_entries():
    rng = np.random.default_rng(101)
    out = []
    n = 1000
    # sign-crossing data: every delta has leading count 0 and, from the first '11' on, every window is 64 bits
    v = np.abs(rng.standard_normal(n // 2)) * np.where(np.arange(n // 2) % 2 == 0, -1.0, 1.0)
    out.append(_full(L.TYPE_FLOAT, "g_sign", _pairs(v), dict(codec="gorilla", leads={0}, leads_within={0}, min_m64=1), tags={"il"}))
    # the longest run of 66-bit '10' records the encoder writes into one page: a 64-bit window opened by the first record
    # (sign and lowest bit flip), then every row a new sign-crossing value; the tail repeats to stay under 90 % of raw
    v = lane_values("dense", rng, n)
    out.append(_full(L.TYPE_FLOAT, "g_dense66", v, dict(codec="gorilla", leads_within={0}, min_m64=1, min_run66=790), tags={"il"}))
    # leading count exactly 1: values alternate across 2.0 (bit 62 flips, the sign never does)
    lo = rng.uniform(0.5, 2.0, n // 2); hi = rng.uniform(2.0, 8.0, n // 2)
    v = np.empty(n); v[0::2] = lo; v[1::2] = hi
    v = np.repeat(v[: n // 2], 2)
    out.append(_full(L.TYPE_FLOAT, "g_lead1", v, dict(codec="gorilla", leads={1}, leads_within={1}), tags={"il"}))
    # leading count exactly 2: random bit patterns below 0x4000.. (positive doubles under 2, subnormals included) with bit 61
    # flipping every value: the edge of k_fused_il's in-place '10' decode
    u = rng.integers(0, 1 << 61, n // 2, dtype=np.uint64) | (np.arange(n // 2, dtype=np.uint64) % np.uint64(2)) << np.uint64(61)
    u[0:40:4] = rng.integers(1, 1 << 52, 10, dtype=np.uint64)  # subnormals (bit 61 clear: the even positions)
    out.append(_full(L.TYPE_FLOAT, "g_lead2", _u2f(np.repeat(u, 2)), dict(codec="gorilla", leads={2}, leads_within={2}), tags={"il"}))
    # leading count exactly 3
    u = np.uint64(1 << 61) | rng.integers(0, 1 << 60, n // 2, dtype=np.uint64) | (np.arange(n // 2, dtype=np.uint64) % np.uint64(2)) << np.uint64(60)
    out.append(_full(L.TYPE_FLOAT, "g_lead3", _u2f(np.repeat(u, 2)), dict(codec="gorilla", leads={3}, leads_within={3}), tags={"il"}))
    # deltas of 34, 33 and 32 leading zeros: the encoder stores clz & 0x1F, so 32 and 33 open windows of stored leading count 0
    # and 1 (and write the full 64 - trailing bits), 34 opens one of 2.  Triples in that order with a trailing count that falls
    # from triple to triple make every one of them open a window
    base = np.uint64(0x412E848000000000)  # 1e6
    ds = []
    for k, tz in enumerate(range(28, -1, -1)):
        for clz in (34, 33, 32):
            top = 63 - clz
            mid = int(rng.integers(0, 1 << max(1, top - tz - 1))) << (tz + 1) if top - tz > 1 else 0
            ds.append((1 << top) | (mid & ((1 << top) - 1)) | (1 << tz))
    while len(ds) < n // 4:
        ds.append((1 << 31) | (int(rng.integers(0, 1 << 31)) | 1))
    u = []
    for dd in ds:  # b, b, b^d, b^d: every delta is a d, half the records are '0'
        u += [int(base), int(base), int(base) ^ dd, int(base) ^ dd]
    out.append(_full(L.TYPE_FLOAT, "g_wrap", _u2f(u[:n]), dict(codec="gorilla", lead_pairs={(0, 32), (1, 33), (2, 34)}), tags={"il"}))
    out.append(_full(L.TYPE_FLOAT, "g_switch", lane_values("switch", rng, n), dict(codec="gorilla", leads={0, 2}, min_lead_switches=10), tags={"il"}))
    # (almost) only '0' records: ten values in runs of 100 (a page of one value is Same, of <= 8 values RLE)
    v = np.repeat(rng.standard_normal(10) + 100, n // 10)
    out.append(_full(L.TYPE_FLOAT, "g_zeros", v, dict(codec="gorilla", min_zero_frac=0.99), tags={"il"}))
    # special values, one infinity sign per page (the encoder refuses a page whose running sum meets both: +-DBL_MAX come in
    # pairs that cancel)
    for sign, nm in ((1.0, "g_special_pinf"), (-1.0, "g_special_ninf")):
        v = _pairs(rng.standard_normal(n // 2) * 10)
        v[10:12] = 0.0; v[20:22] = -0.0; v[30:32] = 5e-324; v[40:42] = -2.5e-310; v[50:52] = (DBL_MAX, -DBL_MAX); v[60:62] = (-DBL_MAX, DBL_MAX)
        v[70:72] = sign * np.inf; v[80:82] = 2.2250738585072014e-308
        out.append(_full(L.TYPE_FLOAT, nm, v, dict(codec="gorilla"), tags={"il", "inf"}))
    # other codecs
    u = rng.integers(0, 1 << 62, n, dtype=np.uint64) | np.uint64(1 << 62)
    u = np.where((u >> np.uint64(52)) & np.uint64(0x7FF) == np.uint64(0x7FF), np.uint64(0x4000000000000000), u)
    out.append(_full(L.TYPE_FLOAT, "f_raw", _u2f(u), dict(codec="raw"), tags={"il"}))
    v = rng.standard_normal(n); v[rng.integers(0, n, 60)] = np.nan; v[0] = np.nan; v[999] = np.nan
    page = np.concatenate([np.frombuffer(struct.pack(">BIB", 31, n, 0x00), np.uint8), v.view(np.uint8)])
    out.append(Entry("f_raw_nan", L.TYPE_FLOAT, v, np.ones(n, bool), page, dict(codec="raw", header="full"), encoder_built=False,
                     twin=[_fpage(v)], note="the encoder writes NaN raw only for segments of <= 4 rows and picks Snappy otherwise",
                     tags={"il", "nan"}))
    out.append(_full(L.TYPE_FLOAT, "f_same", np.full(n, 3.25), dict(codec="same")))
    out.append(_full(L.TYPE_FLOAT, "f_same0", np.zeros(n), dict(codec="same")))
    out.append(_full(L.TYPE_FLOAT, "f_rle", np.repeat([1.5, 0.0, -7.0, 0.0, 2.0**-1074, -3.0], [200, 100, 300, 50, 250, 100]),
                     dict(codec="rle", min_rle_zero_runs=2)))
    big = np.concatenate([np.full(16384 + 16383, 4.5), np.zeros(16384 + 5), np.full(3, -1.0)])
    out.append(_full(L.TYPE_FLOAT, "f_rle_cap", big, dict(codec="rle", min_rle_zero_runs=2, min_rle_max_run=16384), tags={"long"}))
    out.append(_full(L.TYPE_FLOAT, "f_one", np.array([-42.5]), dict(header="one", codec="one")))
    e = _full(L.TYPE_FLOAT, "f_empty", np.zeros(n), dict(header="empty", codec="empty"))
    e.valid[:] = False; e.page = _fpage(e.cells, e.valid.astype(np.uint8))
    out.append(e)
    return out


def int_entries():
    rng = np.random.default_rng(202)
    n = 1000
    out = [_full(L.TYPE_INT, "i_const_pos", np.arange(n, dtype=np.int64) * 7 - 3500, dict(codec="const")),
           _full(L.TYPE_INT, "i_const_neg", np.arange(n, dtype=np.int64) * -123456789 + 10**9, dict(codec="const")),
           _full(L.TYPE_INT, "i_const_zero", np.full(n, -77, np.int64), dict(codec="const"))]
    # every Simple8b selector: a group of n_s zig-zag deltas for s = 2..15 whose first needs exactly bits_s bits (so no earlier
    # selector fits), twice; then a tail of 360 steps of -1 (zig-zag 1): selectors 0 and 1, 240 + 120 ones, which canPack takes
    # only when every remaining value is 1
    zz = []
    for _rep in range(2):
        for s in range(2, 16):
            cnt, bits = S8B_TABLE[s]
            zz += [(1 << bits) - 1] + [int(x) for x in rng.integers(0, 1 << bits, cnt - 1, dtype=np.uint64)]
    zz += [1] * 360
    deltas = [(z >> 1) ^ -(z & 1) for z in zz]
    v = np.cumsum(np.array([5] + deltas, dtype=object)).astype(np.int64)
    out.append(_full(L.TYPE_INT, "i_s8b_all", v, dict(codec="s8b", selectors=set(range(16)))))
    # a tail of exactly 240 ones (one selector-0 word) and of exactly 120 (one selector-1 word): a decoder that swaps the two
    # runs out of words, or stops inside one
    for k, sel in ((240, 0), (120, 1)):
        zz = [int(x) for x in rng.integers(0, 1 << 12, 100)] + [1] * k
        v = np.cumsum(np.array([3] + [(z >> 1) ^ -(z & 1) for z in zz], dtype=object)).astype(np.int64)
        out.append(_full(L.TYPE_INT, f"i_s8b_tail{k}", v, dict(codec="s8b", selectors={sel})))
    # values near +-2^62: deltas are small (Simple8b), sums wrap int64
    out.append(_full(L.TYPE_INT, "i_s8b_hi", (1 << 62) + np.cumsum(rng.integers(-1000, 1001, n)).astype(np.int64), dict(codec="s8b")))
    out.append(_full(L.TYPE_INT, "i_s8b_lo", -(1 << 62) - np.cumsum(rng.integers(0, 5000, n)).astype(np.int64), dict(codec="s8b")))
    out.append(_full(L.TYPE_INT, "i_near53", (1 << 53) + np.cumsum(rng.integers(-3, 4, n)).astype(np.int64), dict(codec="s8b")))
    out.append(_full(L.TYPE_INT, "i_raw2",np.array([I64_MIN, I64_MAX], np.int64), dict(codec="raw")))
    v = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    v[0], v[1], v[500], v[999] = I64_MIN, I64_MAX, I64_MIN, I64_MAX
    zz = (v.astype(np.uint64) << np.uint64(1)) ^ (v >> np.int64(63)).astype(np.uint64)
    page = np.concatenate([np.frombuffer(struct.pack(">BIBI", 32, n, 0x40, 8 * n), np.uint8), zz.astype(">u8").view(np.uint8)])
    out.append(Entry("i_raw", L.TYPE_INT, v, np.ones(n, bool), page, dict(codec="raw", header="full"), encoder_built=False,
                     twin=[oracle.field_page_encode(L.TYPE_INT, v[i:i + 2]) for i in range(0, n, 2)],
                     note="the encoder writes raw int blocks only for fewer than 3 values (zstd otherwise, not restated)"))
    out.append(_full(L.TYPE_INT, "i_one", np.array([I64_MIN], np.int64), dict(header="one", codec="one")))
    e = _full(L.TYPE_INT, "i_empty", np.zeros(n, np.int64), dict(header="empty", codec="empty"))
    e.valid[:] = False; e.page = oracle.field_page_encode(L.TYPE_INT, e.cells, np.zeros(n, np.uint8))
    out.append(e)
    return out


def bool_entries():
    rng = np.random.default_rng(303)
    n = 1000
    out = [_full(L.TYPE_BOOL, "b_full", (rng.random(n) < 0.5).astype(np.uint8), dict(codec="bits", header="full")),
           _full(L.TYPE_BOOL, "b_one", np.array([1], np.uint8), dict(header="one", codec="one"))]
    e = _full(L.TYPE_BOOL, "b_empty", np.zeros(n, np.uint8), dict(header="empty", codec="empty"))
    e.valid[:] = False; e.page = oracle.field_page_encode(L.TYPE_BOOL, e.cells, np.zeros(n, np.uint8))
    out.append(e)
    return out


def with_nulls(e, seed):
    """The entry with null rows.  Nulls are inserted between the values, so the block (and every form it holds) stays the same,
    as long as the page stays within 1000 rows (the segment size of the reference writer, and what k_fused_cols and
    og_encode_pages take); a 1000-row entry instead loses k of its values, to keep 1000 rows"""
    rng = np.random.default_rng(seed)
    k = max(3, e.rows // 7)
    vals = e.cells
    forms = {k2: v for k2, v in e.forms.items() if k2 != "header"}
    if 1000 < e.rows + k and e.rows <= 1000:
        if forms.get("codec") in ("const", "same", "rle") or "min_zero_frac" in forms:  # runs and steps survive a cut tail
            vals = e.cells[:e.rows - k]
        else:  # dense streams keep their mix of records when the k values go from all over the page
            vals = np.delete(e.cells, np.sort(rng.choice(np.arange(1, e.rows - 1), k, replace=False)))
        if "min_run66" in forms:
            forms["min_run66"] = int(forms["min_run66"] * vals.size / e.rows * 0.95)
    rows = vals.size + k
    valid = np.ones(rows, bool)
    valid[rng.choice(np.arange(1, rows - 1), k, replace=False)] = False
    cells = np.zeros(rows, e.cells.dtype)
    cells[valid] = vals
    if e.encoder_built:
        page = oracle.field_page_encode(e.typ, cells, valid.astype(np.uint8))
    else:  # the hand-built raw block of the kept values under a hand-built normal header (EncodeColumnHeader)
        if e.typ == L.TYPE_FLOAT:
            block = np.concatenate([np.zeros(1, np.uint8), vals.astype("<f8").view(np.uint8)])
        else:
            zz = (vals.astype(np.uint64) << np.uint64(1)) ^ (vals >> np.int64(63)).astype(np.uint64)
            block = np.concatenate([np.frombuffer(struct.pack(">BI", 0x40, 8 * vals.size), np.uint8), zz.astype(">u8").view(np.uint8)])
        bm = np.packbits(valid.astype(np.uint8), bitorder="little")
        page = np.concatenate([np.array([e.typ], np.uint8), np.frombuffer(struct.pack(">I", bm.size), np.uint8), bm,
                               np.frombuffer(struct.pack(">II", 0, k), np.uint8), block])
    forms["header"] = "normal"
    return Entry(e.name + "_nulls", e.typ, cells, valid, page, forms, twin=None, encoder_built=e.encoder_built,
                 note=e.note, tags=set(e.tags) | {"nulls"})


def with_bm_off(e, off, seed):
    """A column sliced from a record keeps BitMapOffset & 7 in its header (subBitmapBytes): the validity bit of row i sits at
    bit off + i, and the bits below it belong to rows before the slice.  Every encoder here writes 0, so the header is
    rewritten by hand; the bits below the offset are random"""
    h = read_header(e.page)
    assert h["kind"] == "normal" and h["bm_off"] == 0
    rows = e.rows
    bits = np.zeros(off + rows, np.uint8)
    bits[:off] = np.random.default_rng(seed).integers(0, 2, off)
    bits[off:] = e.valid
    bm = np.packbits(bits, bitorder="little")
    page = np.concatenate([e.page[:1], np.frombuffer(struct.pack(">I", bm.size), np.uint8), bm,
                           np.frombuffer(struct.pack(">II", off, h["nil"]), np.uint8), h["block"]])
    forms = dict(e.forms, bm_off=off)
    return Entry(f"{e.name}_bmoff{off}", e.typ, e.cells, e.valid, page, forms, twin=[e.page], encoder_built=False,
                 note="every encoder writes a bitmap offset of 0", tags=set(e.tags) | {"bm_off"})


def value_entries():
    """every float, int and bool entry, each also with nulls, and the null variants of a few with bm_off 1..7"""
    base = float_entries() + int_entries() + bool_entries()
    out = list(base)
    nulls = {}
    for i, e in enumerate(base):
        if e.forms.get("header") in ("one", "empty"):
            continue
        ne = with_nulls(e, 1000 + i)
        out.append(ne)
        nulls[e.name] = ne
    for off, name in zip(range(1, 8), ["g_sign", "i_s8b_all", "b_full", "f_rle", "i_const_neg", "f_same", "g_lead2"]):
        out.append(with_bm_off(nulls[name], off, off))
    return out


def time_entries():
    rng = np.random.default_rng(404)
    out = []

    def t(name, times, forms, **kw):
        times = np.asarray(times, np.int64)
        return Entry(name, TIME, times, np.ones(times.size, bool), oracle.time_page_encode(times), forms, **kw)
    out.append(t("t_const", T0 + np.arange(1000, dtype=np.int64) * SEC, dict(codec="t_const")))
    out.append(t("t_s8b_scaled", T0 + np.cumsum(rng.integers(1, 50, 1000) * 1_000_000).astype(np.int64), dict(codec="t_s8b", scale=1_000_000)))
    out.append(t("t_s8b_unscaled", T0 + 1 + np.cumsum(rng.integers(1, 5000, 777)).astype(np.int64), dict(codec="t_s8b", scale=1)))
    out.append(t("t_raw2", [T0, T0 + 17], dict(codec="t_raw")))
    out.append(t("t_one", [T0 + 5], dict(codec="t_one")))
    out.append(t("t_pre1970", -5_000_000 * SEC + np.arange(1000, dtype=np.int64) * SEC, dict(codec="t_const"), tags={"negative"}))
    out.append(t("t_cross0", -500 * SEC + 3 + np.arange(1000, dtype=np.int64) * SEC, dict(codec="t_const"), tags={"negative", "nan_times"}))
    out.append(t("t_nan_doubles", -(1 << 52) + 7 + np.arange(1000, dtype=np.int64) * (SEC // 10), dict(codec="t_const"),
                 tags={"negative", "nan_times"}))
    out.append(t("t_pre1970_s8b", -3_000_000 * SEC + np.cumsum(rng.integers(1, 50, 1000) * SEC).astype(np.int64),
                 dict(codec="t_s8b", scale=SEC), tags={"negative"}))
    return out
