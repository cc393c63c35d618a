"""An INDEPENDENT second encoder for openGemini's column page wire format, written in plain Python straight from the Go sources
(not from oracle/): it exists to pin the oracle's encoders/decoders — and through them the GPU decoders — against a second
reading of the reference, since the reference ships no golden bytes (SURVEY §8c).

Sources restated (paths in /root/reference):
  lib/util/lifted/influxdb/tsdb/engine/tsm1/batch_float.go:17-254   FloatArrayEncodeAll (Gorilla; leading &= 0x1F quirk)
  lib/compress/float.go:60-101,171-262                                adaptive float selection (raw / same / RLE / gorilla; Snappy not restated)
  lib/compress/compress.go:38-93                                      SameValueEncoding, RLE.Encoding
  lib/encoding/int.go:66-212                                          Integer.Encoding (const-delta / simple8b / raw)
  lib/util/lifted/encoding/simple8b/encoding.go:350-473               EncodeAll, canPack (selector 0/1 quirk: ALL remaining == 1)
  lib/encoding/timestamp.go:34-190                                    Time.Encoding (const-delta / simple8b + scale / raw)
  lib/encoding/bool.go:40-61                                          Boolean.Encoding (MSB-first bit pack)
  engine/immutable/column_builder.go:428-502                          EncodeColumnHeader / one-row mode / Full / Empty rewrite
Everything is done with Python ints and a list of bits: slow, obviously correct, no shared code with the C++ oracle.
"""
import math
import struct

M64 = (1 << 64) - 1
UVNAN = 0x7FF8000000000001
S8B_MAX = (1 << 60) - 1
S8B = [(240, 0), (120, 0), (60, 1), (30, 2), (20, 3), (15, 4), (12, 5), (10, 6), (8, 7), (7, 8), (6, 10), (5, 12), (4, 15), (3, 20), (2, 30), (1, 60)]


def f2u(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def uvarint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def zigzag(v):
    return ((v << 1) ^ (v >> 63)) & M64


class Bits:
    def __init__(self):
        self.b = []

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.b.append((v >> i) & 1)

    def bytes(self):
        pad = (-len(self.b)) % 8
        bits = self.b + [0] * pad
        return bytes(int("".join(map(str, bits[i:i + 8])), 2) for i in range(0, len(bits), 8))


def gorilla(values):
    """FloatArrayEncodeAll: [0x10][first 8 B BE][records...][NaN sentinel record]; length = ceil(bits / 8)."""
    if values and math.isnan(values[0]):
        raise ValueError("unsupported value: NaN")
    w = Bits()
    w.put(0x10, 8)
    rest = list(values[1:])
    prev = f2u(values[0]) if values else UVNAN
    w.put(prev, 64)
    finished = not values
    prev_lead, prev_trail = None, 0
    i = 0
    total = 0.0
    while not finished:
        if i < len(rest):
            x = rest[i]; total += x; cur = f2u(x)
        else:
            cur = UVNAN; finished = True
        i += 1
        d = cur ^ prev
        if d == 0:
            w.put(0, 1); prev = cur
            continue
        w.put(1, 1)
        lead = (64 - d.bit_length()) & 0x1F          # clz & 0x1F: 32 wraps to 0; the ">= 32 -> 31" clamp after it is dead code
        trail = (d & -d).bit_length() - 1
        if prev_lead is not None and lead >= prev_lead and trail >= prev_trail:
            w.put(0, 1)
            l = 64 - prev_lead - prev_trail
            w.put((d >> prev_trail) & ((1 << l) - 1), l)
        else:
            prev_lead, prev_trail = lead, trail
            w.put(1, 1)
            w.put(lead, 5)
            sig = 64 - lead - trail
            w.put(sig & 0x3F, 6)                       # 64 is written as 0
            w.put((d >> trail) & ((1 << sig) - 1), sig)
        prev = cur
    if math.isnan(total):
        raise ValueError("unsupported value: NaN")
    return w.bytes()


def _is_int(f):
    if 0 <= f < (1 << 32):
        return float(int(f)) == f
    if math.isinf(f):                                   # Go: math.Ceil(+-Inf) == +-Inf (Python's math.ceil raises)
        return True
    return math.ceil(f) == f and math.floor(f) == f


def float_block(values):
    """Float.adaptiveEncoding; returns None where the reference would call Snappy (third-party bytes, not restated)."""
    n = len(values)
    raw = b"\x00" + struct.pack("<%dd" % n, *values)
    if n <= 4:
        return raw
    distinct = 1 + sum(1 for i in range(1, n) if values[i] != values[i - 1])   # float compare, like the Go code
    extreme = any(math.isnan(v) for v in values)
    if distinct == 1:
        out = b"\x40" + struct.pack(">H", n & 0xFFFF)
        return out if values[0] == 0 else out + struct.pack("<d", values[0])
    if distinct <= 8:
        out = bytearray(b"\x50")
        u = [f2u(v) for v in values]
        run = 1
        for i in range(1, n + 1):
            if i < n and u[i] == u[i - 1] and run < (1 << 14):
                run += 1
                continue
            if u[i - 1] == 0:
                out += struct.pack(">H", run | (1 << 15))
            else:
                out += struct.pack(">H", run) + struct.pack("<Q", u[i - 1])
            run = 1
        return bytes(out)
    k = less = 0
    int_only = True
    for v in values:
        if k >= n // 10:
            break
        if v == 0:
            continue
        k += 1
        if int_only and not _is_int(v):
            int_only = False
        if _is_int(v * 1000):
            less += 1
    less_decimal = k > 0 and (100 * less // k) > 90
    if (not int_only and less_decimal) or extreme:
        return None
    out = b"\x30" + gorilla(values)
    if len(out) > n * 8 * 90 // 100:
        return raw
    return out


def s8b_encode_all(src):
    words, i = [], 0
    while i < len(src):
        rem = src[i:]
        for sel, (n, bits) in enumerate(S8B):
            if len(rem) < n:
                continue
            if bits == 0:
                ok = all(v == 1 for v in rem)            # canPack quirk: every REMAINING value must be 1
            else:
                ok = all(v <= (1 << bits) - 1 for v in rem[:n])
            if ok:
                w = sel << 60
                if bits:
                    for k in range(n):
                        w |= rem[k] << (k * bits)
                words.append(w); i += n
                break
        else:
            raise ValueError("value out of bounds")
    return words


def int_block(values):
    n = len(values)
    raw = lambda: b"\x40" + struct.pack(">I", 8 * n) + b"".join(struct.pack(">Q", zigzag(v)) for v in values)
    if n < 3:
        return raw()
    zz = [zigzag(values[0])] + [zigzag(values[i] - values[i - 1]) for i in range(1, n)]
    is_const = all(zz[i - 1] == zz[i] for i in range(2, n))
    is_s8b = all(z <= S8B_MAX for z in zz[1:])
    if is_const:
        return b"\x10" + struct.pack(">Q", zz[0]) + uvarint(zz[1]) + uvarint(n - 1)
    if is_s8b:
        words = s8b_encode_all(zz[1:])
        return b"\x20" + struct.pack(">II", len(words) + 1, n) + struct.pack(">Q", zz[0]) + b"".join(struct.pack(">Q", w) for w in words)
    return None  # zstd: third-party, not restated


def time_block(times):
    n = len(times)
    t = [x & M64 for x in times]
    if n < 3:
        return b"\x40" + struct.pack(">I", 8 * n) + b"".join(struct.pack(">Q", zigzag(x)) for x in times)
    deltas = [t[0]] + [(t[i] - t[i - 1]) & M64 for i in range(1, n)]
    sc = 1
    for s in (10 ** k for k in range(12, 0, -1)):
        if deltas[n - 1] % s == 0:
            sc = s
            break
    is_const, is_s8b = True, deltas[n - 1] < S8B_MAX
    for i in range(n - 2, 0, -1):
        while sc > 1 and deltas[i] % sc != 0:
            sc //= 10
        is_const = is_const and deltas[i] == deltas[i + 1]
        is_s8b = is_s8b and deltas[i] < S8B_MAX
    if is_const:
        return b"\x10" + struct.pack(">Q", deltas[0]) + uvarint(deltas[1]) + uvarint(n - 1)
    if is_s8b:
        words = s8b_encode_all([d // sc for d in deltas[1:]])
        return b"\x20" + struct.pack(">Q", sc) + struct.pack(">II", len(words) + 1, n) + struct.pack(">Q", deltas[0]) + b"".join(struct.pack(">Q", w) for w in words)
    return None  # snappy


def bool_block(values):
    w = Bits()
    for v in values:
        w.put(1 if v else 0, 1)
    return b"\x10" + struct.pack(">I", len(values)) + w.bytes()


TYPE_INT, TYPE_FLOAT, TYPE_BOOL = 1, 3, 5


def field_page(typ, cells, valid=None):
    """EncodeColumnHeader + the block of the non-null values.  cells: one per row; valid: None or per-row 0/1."""
    rows = len(cells)
    if valid is None:
        valid = [1] * rows
    vals = [c for c, k in zip(cells, valid) if k]
    nil = rows - len(vals)
    if rows == 1 and len(vals) == 1:                      # CanEncodeOneRowMode: one row whose Val is 1..15 bytes
        body = bytes([1 if vals[0] else 0]) if typ == TYPE_BOOL else (struct.pack("<d", vals[0]) if typ == TYPE_FLOAT else struct.pack("<q", vals[0]))
        return bytes([16 + {TYPE_INT: 2, TYPE_FLOAT: 1, TYPE_BOOL: 3}[typ]]) + body
    block = {TYPE_FLOAT: float_block, TYPE_INT: int_block, TYPE_BOOL: bool_block}[typ](vals) if vals else b""
    if block is None:
        return None
    code = {TYPE_INT: 2, TYPE_FLOAT: 1, TYPE_BOOL: 3}[typ]
    if nil == 0:
        return bytes([30 + code]) + struct.pack(">I", rows) + block
    if nil == rows:
        return bytes([40 + code]) + struct.pack(">I", rows)
    bm = bytearray((rows + 7) // 8)
    for i, k in enumerate(valid):
        if k:
            bm[i >> 3] |= 1 << (i & 7)
    return bytes([typ]) + struct.pack(">I", len(bm)) + bytes(bm) + struct.pack(">II", 0, nil) + block


def time_page(times):
    if len(times) == 1:
        return bytes([18]) + struct.pack("<q", times[0])
    blk = time_block(list(times))
    return None if blk is None else bytes([32]) + struct.pack(">I", len(times)) + blk
