"""Generates tests/golden/jpeg_foreign.npz: JPEG files cv2.imencode did not write (tests/jpeg_foreign_cases.py names them), and
what cv2.imdecode(bytes, IMREAD_COLOR) makes of each: its frame (in full up to jpeg_cases.FULL_BYTES, else its SHA-256), or that
it returned None.  OpenCV and Pillow are present where goldens are generated only, so no test imports them.  The versions go to
tests/golden/META_jpeg_foreign.json.

    python tests/golden/make_golden_jpeg_foreign.py

The files come from four sources:
- Pillow's encoder (its own tables, restart options, ICC / COM segments, grey);
- cv2 files with their headers rewritten (fill bytes, table layout, component ids, APP0 / APP14, EXIF, what follows the scan);
- a small baseline encoder below, which writes chosen tables (16-bit DQT, per-component tables, Huffman codes of chosen lengths)
  and chosen symbol streams (sizes 11-15, ZRL runs ending at or past coefficient 63, extreme coefficients and DC walks);
- cv2 files with seeded damage to the scan (changed bytes, stray markers and FF bytes, RSTn markers dropped / duplicated /
  renumbered, truncation)."""
import heapq
import io
import json
import os
import re
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

NATURAL = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
           62, 63]


# ---- segments of a file ---------------------------------------------------------------------------------------------------------
def seg(m, payload):
    return bytes([0xFF, m]) + struct.pack(">H", len(payload) + 2) + payload


def split(b):
    """([(marker, payload)] from after SOI up to and including SOS, the bytes after SOS's header: scan, EOI and anything else)"""
    out, pos = [], 2
    while True:
        assert b[pos] == 0xFF
        m, n = b[pos + 1], struct.unpack(">H", b[pos + 2:pos + 4])[0]
        out.append((m, b[pos + 4:pos + 2 + n]))
        pos += 2 + n
        if m == 0xDA:
            return out, b[pos:]


def join(segs, rest):
    return b"\xff\xd8" + b"".join(seg(m, p) for m, p in segs) + rest


def scan_bytes(rest):
    """The entropy-coded data of `rest` (split's second part): up to its last FF D9."""
    return rest[:rest.rindex(b"\xff\xd9")]


# ---- a baseline encoder ---------------------------------------------------------------------------------------------------------
class Table:
    """A Huffman table from (symbol, code length) pairs: the DHT counts and values, and each symbol's canonical code."""

    def __init__(self, lengths):
        self.bits = [0] * 17
        self.vals = []
        for l in range(1, 17):
            for s, ll in lengths:
                if ll == l:
                    self.bits[l] += 1
                    self.vals.append(s)
        self.code, c, k = {}, 0, 0
        for l in range(1, 17):
            for _ in range(self.bits[l]):
                self.code[self.vals[k]] = (c, l)
                c += 1
                k += 1
            assert c < (1 << l), "code lengths overflow (or use the all-ones code)"
            c <<= 1

    def dht(self, tc, th):
        return bytes([tc << 4 | th] + self.bits[1:]) + bytes(self.vals)


def optimal(symbols):
    """Huffman code lengths for a symbol sequence, at most 16 bits, with the all-ones code left unused (a dummy symbol takes it)."""
    freq = {}
    for s in symbols:
        freq[s] = freq.get(s, 0) + 1
    heap = [(n, i, [s]) for i, (s, n) in enumerate(sorted(freq.items()))] + [(0, -1, [None])]
    heapq.heapify(heap)
    depth = {s: 0 for s in freq}
    depth[None] = 0
    k = len(heap)
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        for s in a[2] + b[2]:
            depth[s] += 1
        heapq.heappush(heap, (a[0] + b[0], k, a[2] + b[2]))
        k += 1
    if max(depth.values()) > 16:                   # flat fallback: every symbol one length
        L = max(1, int(np.ceil(np.log2(len(freq) + 1))))
        return Table([(s, L) for s in sorted(freq)])
    return Table(sorted(((s, max(d, 1)) for s, d in depth.items() if s is not None), key=lambda t: (t[1], t[0])))


def size(v):
    return int(abs(int(v))).bit_length()


def tokens(zz):
    """One block's AC symbols (run, size, value) from its 64 zigzag-ordered coefficients, EOB as (0, 0, 0), ZRL as (15, 0, 0)."""
    out, run = [], 0
    for k in range(1, 64):
        v = int(zz[k])
        if v == 0:
            run += 1
            continue
        while run > 15:
            out.append((15, 0, 0))
            run -= 16
        out.append((run, size(v), v))
        run = 0
    if run:
        out.append((0, 0, 0))
    return out


class Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, code, n):
        self.acc, self.n = (self.acc << n) | code, self.n + n
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 255
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        return bytes(self.out)


def amplitude(v, s):
    return v if v >= 0 else v + (1 << s) - 1


class Frame:
    """A baseline file being built: comps [(id, h, v, tq)], blocks[c] a [rows][cols] grid of (dc, [AC symbols]) in block units."""

    def __init__(self, w, h, comps, blocks):
        self.w, self.h, self.comps, self.blocks = w, h, comps, blocks
        self.hmax = max(c[1] for c in comps) if len(comps) > 1 else 1
        self.vmax = max(c[2] for c in comps) if len(comps) > 1 else 1
        self.mcux, self.mcuy = -(-w // (8 * self.hmax)), -(-h // (8 * self.vmax))

    def mcu_blocks(self, m):
        mx, my = m % self.mcux, m // self.mcux
        for c, (_, hs, vs, _) in enumerate(self.comps):
            if len(self.comps) == 1:
                hs = vs = 1
            for bv in range(vs):
                for bh in range(hs):
                    yield c, self.blocks[c][my * vs + bv][mx * hs + bh]

    def symbols(self, restart=0):
        """(component, 'dc' | 'ac', symbol, bits, nbits) in scan order, as list per restart interval"""
        out, pred = [[]], [0] * len(self.comps)
        for m in range(self.mcux * self.mcuy):
            if restart and m and m % restart == 0:
                out.append([])
                pred = [0] * len(self.comps)
            for c, (dc, ac) in self.mcu_blocks(m):
                d = dc - pred[c]
                pred[c] = dc
                s = size(d)
                out[-1].append((c, "dc", s, amplitude(d, s) if s else 0, s))
                for r, s, v in ac:
                    out[-1].append((c, "ac", r << 4 | s, amplitude(v, s) if s else 0, s))
        return out

    def encode(self, tables, restart=0):
        """The entropy-coded pieces, one per restart interval; tables[(c, 'dc' | 'ac')] is a Table."""
        pieces = []
        for interval in self.symbols(restart):
            b = Bits()
            for c, kind, sym, bits, n in interval:
                code, l = tables[(c, kind)].code[sym]
                b.put(code, l)
                if n:
                    b.put(bits, n)
            pieces.append(b.flush())
        return pieces

    def file(self, tables, qt, *, restart=0, pq=None, sof=0xC0, app=(), rst=None, jfif=True):
        """The whole file: tables[(c, kind)] (a component's tables share a DHT slot when they are the same object), qt {tq: 64
        natural-order values}, pq {tq: 0 | 1}, rst: the RSTn marker bytes between the pieces (default D0, D1, ...)."""
        slots, dht = {}, b""
        for (c, kind), t in tables.items():
            key = (kind, id(t))
            if key not in slots:
                th = sum(1 for k in slots if k[0] == kind)
                slots[key] = th
                dht += t.dht(kind == "ac", th)
        out = [(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")] if jfif else []
        out += list(app)
        for tq, q in sorted(qt.items()):
            p = (pq or {}).get(tq, 0)
            vals = [q[NATURAL[k]] for k in range(64)]
            out.append((0xDB, bytes([p << 4 | tq]) + (struct.pack(">64H", *vals) if p else bytes(vals))))
        sofp = struct.pack(">BHHB", 8, self.h, self.w, len(self.comps))
        for cid, hs, vs, tq in self.comps:
            sofp += bytes([cid, hs << 4 | vs, tq])
        out.append((sof, sofp))
        out.append((0xC4, dht))
        if restart:
            out.append((0xDD, struct.pack(">H", restart)))
        sos = bytes([len(self.comps)])
        for c, (cid, *_) in enumerate(self.comps):
            sos += bytes([cid, slots[("dc", id(tables[(c, "dc")]))] << 4 | slots[("ac", id(tables[(c, "ac")]))]])
        out.append((0xDA, sos + b"\x00\x3f\x00"))
        pieces = self.encode(tables, restart)
        rst = rst if rst is not None else [0xD0 + (k & 7) for k in range(len(pieces) - 1)]
        scan = pieces[0] + b"".join(bytes([0xFF, r]) + p for r, p in zip(rst, pieces[1:]))
        return join(out, scan + b"\xff\xd9")


def optimal_tables(frame, restart=0, shared=False):
    """One optimal DC and AC table per component (luma / chroma pairs when shared)."""
    group = (lambda c: min(c, 1)) if shared else (lambda c: c)
    syms = {}
    for interval in frame.symbols(restart):
        for c, kind, s, _, _ in interval:
            syms.setdefault((group(c), kind), []).append(s)
    built = {k: optimal(v) for k, v in syms.items()}
    return {(c, kind): built[(group(c), kind)] for c in range(len(frame.comps)) for kind in ("dc", "ac")}


def ycc(bgr):
    """JFIF YCbCr planes (float) of a BGR uint8 image."""
    b, g, r = (bgr[..., i].astype(np.float64) for i in range(3))
    y = 0.299 * r + 0.587 * g + 0.114 * b
    return [y, 128 - 0.168736 * r - 0.331264 * g + 0.5 * b, 128 + 0.5 * r - 0.418688 * g - 0.081312 * b]


def quantised(plane, q, rows, cols):
    """The [rows][cols] grid of (dc, AC symbols) of a float plane, edge-padded, DCT'd and quantised by natural-order q."""
    from scipy.fft import dctn
    h, w = plane.shape
    p = np.pad(plane, ((0, max(0, 8 * rows - h)), (0, max(0, 8 * cols - w))), mode="edge")[:8 * rows, :8 * cols] - 128
    blk = p.reshape(rows, 8, cols, 8).transpose(0, 2, 1, 3)
    coef = np.rint(dctn(blk, axes=(2, 3), norm="ortho").reshape(rows, cols, 64) / np.asarray(q, np.float64)).astype(np.int64)
    return [[(int(coef[r, c, 0]), tokens(coef[r, c, NATURAL])) for c in range(cols)] for r in range(rows)]


def encoded_frame(bgr, sampling, qts, tq=(0, 1, 1), ids=(1, 2, 3)):
    """Frame of an image: sampling (h, v) of luma, chroma 1x1, one quantisation table per component as tq says."""
    h, w = bgr.shape[:2]
    hs, vs = sampling
    comps = [(ids[0], hs, vs, tq[0]), (ids[1], 1, 1, tq[1]), (ids[2], 1, 1, tq[2])]
    f = Frame(w, h, comps, None)
    planes = ycc(bgr)
    blocks = []
    for c, pl in enumerate(planes):
        if c:
            H, W = -(-h // vs), -(-w // hs)
            pad = np.pad(pl, ((0, H * vs - h), (0, W * hs - w)), mode="edge")
            pl = pad.reshape(H, vs, W, hs).mean(axis=(1, 3))
        ch, cv = (hs, vs) if c == 0 else (1, 1)
        blocks.append(quantised(pl, qts[comps[c][3]], f.mcuy * cv, f.mcux * ch))
    f.blocks = blocks
    return f


def std_q(scale):
    """A quantisation table: Annex K's luma table times scale, at least 1."""
    k1 = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87,
          80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92,
          95, 98, 112, 100, 103, 99]
    return [max(1, int(round(v * scale))) for v in k1]


# ---- cases -----------------------------------------------------------------------------------------------------------------------
def cv2_file(cv2, seed, h, w, sampling="420", q=90, rst=0):
    import jpeg_cases as jc
    img = jc.image(seed, h, w)
    params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, rst,
              cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + sampling)]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def pillow_files():
    from PIL import Image
    import jpeg_cases as jc
    out = {}

    def save(name, img, **kw):
        b = io.BytesIO()
        img.save(b, "JPEG", **kw)
        out[name] = b.getvalue()

    rgb = Image.fromarray(jc.image(3001, 45, 70)[..., ::-1].copy())
    for s in (0, 1, 2):
        for q in (5, 50, 95):
            save("pil_sub%d_q%d" % (s, q), rgb, quality=q, subsampling=s)
    rs = np.random.RandomState(3002)
    save("pil_qtables3", rgb, qtables=[list(rs.randint(1, 60, 64)), list(rs.randint(2, 90, 64)), list(rs.randint(1, 255, 64))],
         subsampling=0)
    save("pil_qtables2_420", rgb, qtables=[list(rs.randint(1, 30, 64)), list(rs.randint(1, 40, 64))], subsampling=2)
    save("pil_qtables1", rgb, qtables=[list(rs.randint(3, 20, 64))], subsampling=1)
    save("pil_rst_rows", rgb, quality=85, restart_marker_rows=1)
    save("pil_rst_blocks", rgb, quality=85, restart_marker_blocks=5)
    save("pil_optimize", rgb, quality=80, optimize=True)
    save("pil_smooth", rgb, quality=80, smooth=50)
    icc = bytes((np.arange(70000) * 7 // 13 % 251).astype(np.uint8))
    save("pil_icc_com", rgb, quality=80, icc_profile=icc, comment=b"a COM segment")
    save("pil_grey", rgb.convert("L"), quality=80)
    return out


def encoder_files():
    import jpeg_cases as jc
    out = {}
    img = jc.image(3101, 45, 70)
    rs = np.random.RandomState(3102)
    qts = {0: list(rs.randint(1, 40, 64)), 1: list(rs.randint(1, 80, 64)), 2: list(rs.randint(1, 120, 64))}
    f = encoded_frame(img, (2, 2), qts, tq=(0, 1, 2))
    out["enc_qt_percomp"] = f.file(optimal_tables(f), qts)
    qts = {0: std_q(0.5), 1: std_q(1.0)}
    f = encoded_frame(img, (2, 1), qts)
    out["enc_dqt16_le255"] = f.file(optimal_tables(f), qts, pq={0: 1, 1: 1})
    qts = {0: [min(1023, v * 9) for v in std_q(0.5)], 1: [1023 - v for v in std_q(2.0)]}
    f = encoded_frame(img, (2, 2), qts)
    out["enc_dqt16_1023_sof1"] = f.file(optimal_tables(f), qts, pq={0: 1, 1: 1}, sof=0xC1)
    qts = {0: std_q(0.3), 1: std_q(0.6)}
    big = jc.image(3103, 50, 100)                                   # 4:2:0: 7 MCUs a row
    for r in (3, 5, 9):
        f = encoded_frame(big, (2, 2), qts)
        out["enc_rst%d_of7" % r] = f.file(optimal_tables(f, r, shared=True), qts, restart=r)
    return out


def header_files(cv2):
    out = {}
    base = cv2_file(cv2, 3201, 61, 83)
    segs, rest = split(base)
    out["hdr_plain"] = base
    out["hdr_fill"] = b"\xff\xd8" + b"".join(b"\xff" * (1 + k % 3) + seg(m, p) for k, (m, p) in enumerate(segs)) + \
        scan_bytes(rest) + b"\xff\xff\xff\xd9"
    rbase = cv2_file(cv2, 3202, 61, 83, rst=2)
    rsegs, rrest = split(rbase)
    sc = scan_bytes(rrest)
    out["hdr_fill_rst"] = join(rsegs, re.sub(rb"\xff([\xd0-\xd7])", lambda m: b"\xff\xff\xff" + m.group(1), sc) + b"\xff\xd9")   # fill before RSTn too
    dqt = [p for m, p in segs if m == 0xDB]
    dht = [p for m, p in segs if m == 0xC4]
    others = [(m, p) for m, p in segs if m not in (0xDB, 0xC4)]
    sof = next(k for k, (m, _) in enumerate(others) if m == 0xC0)
    pre, post = others[:sof], others[sof:]                                        # post: SOF, SOS
    tabs_one = [(0xDB, b"".join(dqt)), (0xC4, b"".join(dht))]
    tabs_many = []
    for p in dqt:
        o = 0
        while o < len(p):
            n = 1 + 64 * (1 + (p[o] >> 4))
            tabs_many.append((0xDB, p[o:o + n]))
            o += n
    for p in dht:
        o = 0
        while o < len(p):
            n = 17 + sum(p[o + 1:o + 17])
            tabs_many.append((0xC4, p[o:o + n]))
            o += n
    out["hdr_tables_combined"] = join(pre + tabs_one + post, rest)
    out["hdr_tables_split"] = join(pre + tabs_many + post, rest)
    out["hdr_tables_after_sof"] = join(pre + post[:1] + tabs_many[::-1] + post[1:], rest)
    # a first, different definition of every table, then cv2's: the later one is the one the scan uses
    decoy = []
    for m, p in tabs_many:
        if m == 0xDB:
            decoy.append((m, bytes([p[0]]) + bytes(max(1, v // 2 + 1) for v in p[1:])))
        else:
            n = sum(p[1:17])
            decoy.append((m, p[:17] + bytes(reversed(p[17:17 + n]))))
    out["hdr_tables_redefined"] = join(pre + decoy + post[:1] + tabs_many + post[1:], rest)

    def ids(new, segs=segs, rest=rest):
        s = []
        for m, p in segs:
            p = bytearray(p)
            if m == 0xC0:
                for c in range(3):
                    p[6 + 3 * c] = new[c]
            if m == 0xDA:
                for c in range(3):
                    p[1 + 2 * c] = new[c]
            s.append((m, bytes(p)))
        return s

    out["hdr_ids_012"] = join(ids((0, 1, 2)), rest)
    out["hdr_ids_arbitrary"] = join(ids((200, 7, 42)), rest)
    noapp0 = [(m, p) for m, p in segs if m != 0xE0]
    out["hdr_no_jfif"] = join(noapp0, rest)
    adobe = (0xEE, b"Adobe" + struct.pack(">HHHB", 100, 0, 0, 1))
    out["hdr_adobe1"] = join([adobe] + noapp0, rest)
    out["hdr_adobe1_rgb_ids"] = join([adobe] + [sp for sp in ids(b"RGB") if sp[0] != 0xE0], rest)
    out["hdr_rgb_ids_jfif"] = join(ids(b"RGB"), rest)
    out["hdr_rgb_ids_short_jfif"] = join([(0xE0, b"JFIF\0\x01\x01\0\0")] + [sp for sp in ids(b"RGB") if sp[0] != 0xE0], rest)
    out["hdr_rgb_ids_no_jfif"] = join([sp for sp in ids(b"RGB") if sp[0] != 0xE0], rest)
    out["hdr_garbage_after_eoi"] = base + b"\x00\x01garbage\xff\xd8\xff\xe0" + bytes(range(200))
    out["hdr_no_eoi"] = base[:-2]
    return out


def exif_payload(order, entries, ifd=8, cut=None, count=None):
    """'Exif\\0\\0' + a TIFF header in byte order `order` and IFD0 at `ifd` with entries (tag, type, count, 4 value bytes)."""
    e = "<" if order == "II" else ">"
    tiff = order.encode() + struct.pack(e + "HI", 42, ifd) + b"\x5a" * (ifd - 8)
    tiff += struct.pack(e + "H", len(entries) if count is None else count)
    for tag, typ, cnt, val in entries:
        tiff += struct.pack(e + "HHI", tag, typ, cnt) + val
    tiff += struct.pack(e + "I", 0)
    if cut is not None:
        tiff = tiff[:cut]
    return b"Exif\0\0" + tiff


def value(order, typ, v):
    """4 value bytes of a one-element entry of TIFF type typ in byte order order"""
    e = "<" if order == "II" else ">"
    if typ in (1, 2, 6, 7):
        return struct.pack(e + "B", v & 255) + b"\0\0\0"
    if typ in (3, 8):
        return struct.pack(e + "HH", v & 0xFFFF, 0)
    return struct.pack(e + "I", v)


def exif_files(cv2):
    out = {}
    base = cv2_file(cv2, 3301, 37, 53, sampling="422")
    segs, rest = split(base)

    def put(name, payloads, after_dqt=False):
        app = [(0xE1, p) for p in payloads]
        if after_dqt:
            k = max(i for i, (m, _) in enumerate(segs) if m == 0xDB) + 1
            out[name] = join(segs[:k] + app + segs[k:], rest)
        else:
            out[name] = join(segs[:1] + app + segs[1:], rest)

    for order in ("II", "MM"):
        for typ, tn in ((1, "byte"), (3, "short"), (4, "long"), (7, "undef"), (9, "slong")):
            put("exif_%s_%s_6" % (order, tn), [exif_payload(order, [(0x0112, typ, 1, value(order, typ, 6))])])
        put("exif_%s_long_0x60000" % order, [exif_payload(order, [(0x0112, 4, 1, value(order, 4, 0x60000))])])
        put("exif_%s_count0" % order, [exif_payload(order, [(0x0112, 3, 0, value(order, 3, 6))])])
        for v in (0, 9, 0x0106):
            put("exif_%s_value%d" % (order, v), [exif_payload(order, [(0x0112, 3, 1, value(order, 3, v))])])
        put("exif_%s_ifd_at_20" % order, [exif_payload(order, [(0x0112, 3, 1, value(order, 3, 8))], ifd=20)])
        ents = [(0x010F, 2, 4, b"cam\0"), (0x0110, 2, 4, b"mod\0"), (0x0112, 3, 1, value(order, 3, 5)), (0x011A, 5, 1, value(order, 4, 0))]
        put("exif_%s_third_entry" % order, [exif_payload(order, ents)])
        put("exif_%s_truncated_ifd" % order, [exif_payload(order, ents, cut=10 + 2 * 12 + 6)])
        put("exif_%s_truncated_value" % order, [exif_payload(order, ents, cut=10 + 2 * 12 + 9)])
        for k in (10, 11):                                  # the entry's value word is there, its last 2 bytes are not
            put("exif_%s_truncated_entry_%d" % (order, k), [exif_payload(order, ents, cut=10 + 2 * 12 + k)])
        put("exif_%s_one_entry_truncated" % order, [exif_payload(order, [(0x0112, 3, 1, value(order, 3, 6))], cut=10 + 10)])
        put("exif_%s_count_past_end" % order, [exif_payload(order, [(0x0112, 3, 1, value(order, 3, 7))], count=40)])
        put("exif_%s_two_app1" % order, [exif_payload(order, [(0x0112, 3, 1, value(order, 3, 6))]),
                                          exif_payload(order, [(0x0112, 3, 1, value(order, 3, 3))])])
        xmp = b"http://ns.adobe.com/xap/1.0/\0<x:xmpmeta xmlns:x='adobe:ns:meta/'/>"
        put("exif_%s_xmp_first" % order, [xmp, exif_payload(order, [(0x0112, 3, 1, value(order, 3, 8))])])
        put("exif_%s_after_dqt" % order, [exif_payload(order, [(0x0112, 3, 1, value(order, 3, 6))])], after_dqt=True)
    return out


# ---- hand-built entropy data -------------------------------------------------------------------------------------------------------
def grey_frame(w, h, grid):
    return Frame(w, h, [(1, 1, 1, 0)], [grid])


def lengths_table(syms, scheme):
    """A table over syms whose code lengths follow scheme(i) for the i-th symbol."""
    return Table([(s, scheme(i)) for i, s in enumerate(syms)])


def symbol_sets(f):
    dc, ac = set(), set()
    for interval in f.symbols():
        for c, kind, s, _, _ in interval:
            (dc if kind == "dc" else ac).add(s)
    return sorted(dc), sorted(ac)


def hand_files():
    import jpeg_cases as jc
    out = {}
    q = std_q(0.25)
    img = jc.image(3401, 40, 48)
    f0 = encoded_frame(img, (1, 1), {0: q, 1: q})
    grey = grey_frame(48, 40, quantised(ycc(img)[0], q, 5, 6))

    def with_lengths(name, f, scheme_dc, scheme_ac):
        dc, ac = symbol_sets(f)
        tdc, tac = lengths_table(dc, scheme_dc), lengths_table(ac, scheme_ac)
        tabs = {(c, k): (tdc if k == "dc" else tac) for c in range(len(f.comps)) for k in ("dc", "ac")}
        out[name] = f.file(tabs, {0: q, 1: q} if len(f.comps) > 1 else {0: q})

    with_lengths("huff_9bit", grey, lambda i: 9, lambda i: 9)
    with_lengths("huff_10bit", grey, lambda i: 10, lambda i: 10)
    with_lengths("huff_9_10bit", f0, lambda i: 9 + i % 2, lambda i: 9 + (i // 3) % 2)
    with_lengths("huff_8_9_10bit", f0, lambda i: 8 + i % 3, lambda i: 8 + i % 3)
    with_lengths("huff_16bit", f0, lambda i: 2 if i < 2 else 16, lambda i: 3 if i < 4 else 16)
    with_lengths("huff_15_16bit", grey, lambda i: 1 if i == 0 else 15 + i % 2, lambda i: 1 if i == 0 else 15 + i % 2)
    flat = grey_frame(24, 16, [[(0, [(0, 0, 0)]) for _ in range(3)] for _ in range(2)])
    out["huff_one_symbol"] = flat.file({(0, "dc"): Table([(0, 1)]), (0, "ac"): Table([(0, 1)])}, {0: q})
    flat3 = Frame(16, 16, [(1, 2, 2, 0), (2, 1, 1, 1), (3, 1, 1, 1)],
                  [[[(-40 + 5 * x + y, [(0, 0, 0)]) for x in range(2)] for y in range(2)], [[(30, [(0, 0, 0)])]], [[(-20, [(0, 0, 0)])]]])
    out["huff_one_ac_symbol"] = flat3.file(optimal_tables(flat3), {0: q, 1: q})

    # AC sizes 11..15, ZRL runs ending exactly at coefficient 63 and runs past 63, on q = 1 so the values stay in range
    one = [1] * 64
    blocks = []
    rs = np.random.RandomState(3402)
    for k in range(12):
        s = 11 + k % 5
        v = int(rs.choice([-1, 1]) * rs.randint(1 << (s - 1), 1 << s))
        blocks.append((int(rs.randint(-300, 300)), [(int(rs.randint(0, 16)), s, v), (0, 0, 0)]))
    out["ac_size_11_15"] = grey_frame(96, 8, [blocks]).file(*_opt_grey(grey_frame(96, 8, [blocks]), one))
    zrl = [
        (10, [(0, 3, 5), (15, 0, 0), (15, 0, 0), (15, 0, 0), (14, 2, -3)]),                 # 1 + 16*3 + 15 = 63: the last coefficient
        (-20, [(15, 4, 9), (15, 0, 0), (15, 0, 0), (14, 0, 0)][:3] + [(15, 0, 0)]),        # coefficient 16, ZRL to 32, 48, ZRL ends at 64
        (30, [(0, 2, 2)] * 46 + [(15, 0, 0)]),                                             # 46 coefficients, a ZRL ending at 62 + 1
        (0, [(0, 2, 2)] * 47 + [(15, 0, 0)]),                                              # ... ending exactly at 63
        (5, [(0, 1, 1)] * 59 + [(10, 2, 3)]),                                              # k 60 + 10: past 63 (lands on 63)
        (6, [(0, 1, -1)] * 60 + [(15, 0, 0)]),                                             # ZRL from 61 to past 63
        (7, [(0, 1, 1)] * 62 + [(15, 5, 17)]),                                             # 63 + 15
        (8, [(0, 1, 1)] * 63),                                                             # 63 coefficients, no EOB
    ]
    fz = grey_frame(64, 8, [zrl])
    out["ac_zrl_runs_to_63"] = fz.file(*_opt_grey(fz, std_q(0.1)))

    # extreme blocks: dequantised coefficients past int16, pass-1 values past int16, DC walks far outside the baseline range
    for seed in range(6):
        rs = np.random.RandomState(3500 + seed)
        blocks, dc = [], 0
        for k in range(12):
            toks, kk = [], 0
            kind = k % 4
            n = {0: 3, 1: 12, 2: 0, 3: 6}[kind]
            for _ in range(n):
                r = int(rs.randint(0, 6))
                if kk + r + 1 > 63:
                    break
                kk += r + 1
                s = int(rs.randint(6, 16))
                toks.append((r, s, int(rs.choice([-1, 1]) * rs.randint(1 << (s - 1), 1 << s))))
            if kind == 3:                                                          # row 0 only: the zero-column shortcut
                toks = [(0, s, v) for (_, s, v) in toks[:7]]
            if kk < 63:
                toks.append((0, 0, 0))
            dc = int(rs.randint(-16383, 16384)) if seed % 2 else max(-32767, min(32767, dc + int(rs.randint(-2047, 2048))))
            blocks.append((dc, toks))
        qq = list(rs.randint(1, 256, 64)) if seed < 3 else list(rs.randint(200, 1024, 64))
        f = grey_frame(96, 8, [blocks])
        tabs, _ = _opt_grey(f, qq)
        out["extreme_grey_%d" % seed] = f.file(tabs, {0: qq}, pq={0: 0 if seed < 3 else 1})
    rs = np.random.RandomState(3600)
    for seed in range(2):
        def blk():
            toks = [(int(rs.randint(0, 4)), s, int(rs.choice([-1, 1]) * rs.randint(1 << (s - 1), 1 << s)))
                    for s in rs.randint(4, 14, 5)] + [(0, 0, 0)]
            return (int(rs.randint(-3000, 3000)), toks)
        fc = Frame(32, 16, [(1, 2, 2, 0), (2, 1, 1, 1), (3, 1, 1, 1)],
                   [[[blk() for _ in range(4)] for _ in range(2)], [[blk(), blk()]], [[blk(), blk()]]])
        qts = {0: list(rs.randint(1, 200, 64)), 1: list(rs.randint(1, 200, 64))}
        out["extreme_420_%d" % seed] = fc.file(optimal_tables(fc), qts)
    dconly = grey_frame(64, 8, [[(v, [(0, 0, 0)]) for v in (1023, 1024, 2047, -2048, 4095, -4096, 8191, 30000)]])
    out["extreme_dc_only"] = dconly.file(*_opt_grey(dconly, [8] + [1] * 63))
    walk = grey_frame(64, 8, [[(v, [(0, 0, 0)]) for v in (30000, 60000, 90000, 120000, 100000, 70000, 40000, 10000)]])
    out["extreme_dc_walk"] = walk.file(*_opt_grey(walk, [1] * 64))                # the predictor leaves int16; stored truncated
    return out


def _opt_grey(f, q):
    return optimal_tables(f), {0: q}


# ---- damaged scans -----------------------------------------------------------------------------------------------------------------
def corrupt_files(cv2):
    out = {}
    base = cv2_file(cv2, 3701, 61, 83)
    segs, rest = split(base)
    sc = scan_bytes(rest)
    for seed in range(8):
        rs = np.random.RandomState(3710 + seed)
        b = bytearray(sc)
        ok = [i for i in range(1, len(b) - 1) if b[i] != 0xFF and b[i - 1] != 0xFF]
        for i in rs.choice(ok, 3, replace=False):
            b[i] = int(rs.choice([v for v in range(255) if v != b[i]]))
        out["corrupt_bytes_%d" % seed] = join(segs, bytes(b) + b"\xff\xd9")
    mid = [i for i in range(len(sc) // 2, len(sc) - 1) if sc[i - 1] != 0xFF and sc[i] != 0xFF][0]
    for name, marker in (("ff01", b"\xff\x01"), ("ffc4", b"\xff\xc4\x00\x03\x00"), ("ffe0", b"\xff\xe0\x00\x02"),
                         ("ffd9", b"\xff\xd9"), ("ffd0", b"\xff\xd0")):
        out["corrupt_marker_%s" % name] = join(segs, sc[:mid] + marker + sc[mid:] + b"\xff\xd9")   # a stray marker inside the scan
    for seed in range(3):
        rs = np.random.RandomState(3720 + seed)
        b = bytearray(sc)
        ok = [i for i in range(1, len(b) - 1) if b[i] != 0xFF and b[i - 1] != 0xFF]
        for i in rs.choice(ok, 2, replace=False):
            b[i] = 0xFF                                                   # FF followed by whatever byte was there
        out["corrupt_ff_written_%d" % seed] = join(segs, bytes(b) + b"\xff\xd9")
    rbase = cv2_file(cv2, 3702, 61, 83, rst=2)                    # 24 MCUs, 12 intervals, RST0..RST7, RST0..RST2
    rsegs, rrest = split(rbase)
    sc = scan_bytes(rrest)
    marks = [i for i in range(len(sc) - 1) if sc[i] == 0xFF and 0xD0 <= sc[i + 1] <= 0xD7]
    assert len(marks) == 11

    def edit(name, k, new):
        i = marks[k]
        out[name] = join(rsegs, sc[:i] + new + sc[i + 2:] + b"\xff\xd9")

    edit("rst_dropped_3", 3, b"")
    edit("rst_dropped_last", 10, b"")
    edit("rst_duplicated_3", 3, sc[marks[3]:marks[3] + 2] * 2)
    for d in (1, 2, 3, 4, 5, 6, 7):
        edit("rst_renumbered_5_plus%d" % d, 5, bytes([0xFF, 0xD0 + (5 + d) % 8]))
    out["rst_extra_past_last"] = join(rsegs, sc + b"\xff\xd3" + b"\x12\x34" + b"\xff\xd9")
    out["rst_extra_empty_past_last"] = join(rsegs, sc + b"\xff\xd3\xff\xd9")
    cut = rbase
    full = len(cut)
    start = len(join(rsegs, b""))
    for frac in (0.1, 0.5, 0.97):
        out["cut_scan_%d" % int(frac * 100)] = cut[:start + int((full - start) * frac)]
    big = cv2_file(cv2, 3703, 64, 96, q=95)
    ff = big.index(b"\xff\x00", len(join(split(big)[0], b"")))
    out["cut_inside_ff00"] = big[:ff + 1]
    out["cut_after_ff00"] = big[:ff + 2]
    out["cut_before_eoi_ff"] = big[:-1]
    return out


def main():
    import cv2
    import PIL
    import jpeg_cases as jc
    import jpeg_foreign_cases as fc
    files = {}
    files.update(pillow_files())
    files.update(encoder_files())
    files.update(header_files(cv2))
    files.update(exif_files(cv2))
    files.update(hand_files())
    files.update(corrupt_files(cv2))
    assert sorted(files) == sorted(fc.CASES), sorted(set(files) ^ set(fc.CASES))
    out = {}
    for name in fc.CASES:
        buf = np.frombuffer(files[name], np.uint8)
        out["jpg_" + name] = buf
        dec = cv2.imdecode(buf, cv2.IMREAD_COLOR)
        if dec is None:
            out["none_" + name] = np.ones(1, np.uint8)
            continue
        out["shape_" + name] = np.array(dec.shape, np.int64)
        out["sha_" + name] = jc.digest(dec)
        if dec.nbytes <= jc.FULL_BYTES:
            out["bgr_" + name] = dec
    np.savez_compressed(os.path.join(HERE, "jpeg_foreign.npz"), **out)
    meta = {"generator": "tests/golden/make_golden_jpeg_foreign.py", "opencv": cv2.__version__, "pillow": PIL.__version__,
            "libjpeg_turbo": "3.1.2 (OpenCV's bundled build-libjpeg-turbo, x86-64 SIMD: the AVX2 jsimd_idct_islow)",
            "numpy": np.__version__, "cases": len(fc.CASES), "cv2_none": sorted(n for n in fc.CASES if "none_" + n in out)}
    with open(os.path.join(HERE, "META_jpeg_foreign.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    print("wrote %d cases (%d that cv2 cannot decode), %d bytes" % (
        len(fc.CASES), len(meta["cv2_none"]), os.path.getsize(os.path.join(HERE, "jpeg_foreign.npz"))))


if __name__ == "__main__":
    main()
