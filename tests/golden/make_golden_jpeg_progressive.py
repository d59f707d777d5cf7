"""Generates tests/golden/jpeg_progressive.npz: progressive JPEG files (tests/jpeg_progressive_cases.py names them) and what
cv2.imdecode(bytes, IMREAD_COLOR) makes of each, in the format of jpeg_foreign.npz: "jpg_<name>" and either "none_<name>" or
"shape_" / "sha_" and, up to jpeg_cases.FULL_BYTES, "bgr_".  OpenCV and Pillow are present where goldens are generated only.  The
versions go to tests/golden/META_jpeg_progressive.json.

    python tests/golden/make_golden_jpeg_progressive.py

The files come from:
- cv2.imencode with IMWRITE_JPEG_PROGRESSIVE (libjpeg's default script: 10 scans, 6 for grey) and Pillow's progressive=True;
- the reference's two photos re-coded losslessly as progressive files: a small baseline decoder below reads their coefficients,
  and the encoder writes them with cv2's script and with a seeded one (cv2's frames equal frames_modelzoo.npz's, which the
  generator asserts);
- a small progressive encoder below, on the Table / Bits / optimal pieces of make_golden_jpeg_foreign.py, which writes seeded
  scripts of all four scan kinds (1-wide bands, band 63 alone, DC and AC approximation chains from Al up to 13, AC refinement
  over narrow and 1-wide bands, DC interleaved over all, two or one of three components), DRI changed between scans, EOB runs
  past a segment's end, EOB14, ZRL in refinement;
- cv2 progressive files with their scans rewritten: tables redefined, selectors dropped, refinement symbols of size 2, scans dropped,
  moved or with bad parameters, and damage (cuts, changed bytes, RSTn renumbered)."""
import io
import json
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden_jpeg_foreign import NATURAL, Bits, Table, amplitude, optimal, seg, size, ycc  # noqa: E402

PHOTOS = ("000004", "000139")
SCALE = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80,
         62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98,
         112, 100, 103, 99]


# ---- a progressive file as parts ------------------------------------------------------------------------------------------------
def parts(b):
    """[(marker, payload, data)] of a file from after SOI up to EOI; data is a scan's entropy-coded bytes (RSTn included)."""
    out, pos = [], 2
    while True:
        assert b[pos] == 0xFF, pos
        m = b[pos + 1]
        if m == 0xD9:
            return out
        n = struct.unpack(">H", b[pos + 2:pos + 4])[0]
        payload, pos = b[pos + 4:pos + 2 + n], pos + 2 + n
        data = b""
        if m == 0xDA:
            e = pos
            while True:
                e = b.index(b"\xff", e)
                if b[e + 1] == 0 or 0xD0 <= b[e + 1] <= 0xD7:
                    e += 2
                    continue
                break
            data, pos = b[pos:e], e
        out.append((m, payload, data))


def build(ps, eoi=True):
    return b"\xff\xd8" + b"".join(seg(m, p) + d for m, p, d in ps) + (b"\xff\xd9" if eoi else b"")


def scan_indices(ps):
    return [i for i, p in enumerate(ps) if p[0] == 0xDA]


def sos(comps, ss, se, ah, al):
    """A SOS payload: comps [(id, td, ta)]"""
    return bytes([len(comps)] + [v for c in comps for v in (c[0], c[1] << 4 | c[2])] + [ss, se, ah << 4 | al])


def with_sos(ps, k, **kw):
    """ps with scan k's header fields (ss, se, ah, al) replaced"""
    i = scan_indices(ps)[k]
    m, p, d = ps[i]
    ns = p[0]
    f = {"ss": p[1 + 2 * ns], "se": p[2 + 2 * ns], "ah": p[3 + 2 * ns] >> 4, "al": p[3 + 2 * ns] & 15}
    f.update(kw)
    p = p[:1 + 2 * ns] + bytes([f["ss"], f["se"], f["ah"] << 4 | f["al"]])
    return ps[:i] + [(m, p, d)] + ps[i + 1:]


# ---- a progressive encoder (DC first, DC refinement, AC first) ------------------------------------------------------------------
class Coefs:
    """Quantised coefficients of an image: comps [(id, h, v, tq)], coef[c] an int [bh][bw][64] natural-order array over the
    MCU-padded block grid, q {tq: 64 natural-order values}."""

    def __init__(self, bgr, sampling, qs, grey=False):
        from scipy.fft import dctn
        h, w = bgr.shape[:2]
        self.w, self.h = w, h
        hs, vs = (1, 1) if grey else sampling
        self.comps = [(1, 1, 1, 0)] if grey else [(1, hs, vs, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
        self.hmax, self.vmax = hs, vs
        self.mcux, self.mcuy = -(-w // (8 * hs)), -(-h // (8 * vs))
        self.q = {0: qs[0]} if grey else {0: qs[0], 1: qs[1]}
        planes = ycc(bgr)[:1] if grey else ycc(bgr)
        self.coef, self.dw, self.dh = [], [], []
        for c, pl in enumerate(planes):
            ch, cv = self.comps[c][1:3]
            if ch < hs or cv < vs:
                fh, fv = hs // ch, vs // cv
                H, W = -(-h // fv), -(-w // fh)
                pl = np.pad(pl, ((0, H * fv - h), (0, W * fh - w)), mode="edge").reshape(H, fv, W, fh).mean(axis=(1, 3))
            self.dh.append(-(-h * cv // vs))
            self.dw.append(-(-w * ch // hs))
            rows, cols = self.mcuy * cv, self.mcux * ch
            p = np.pad(pl, ((0, max(0, 8 * rows - pl.shape[0])), (0, max(0, 8 * cols - pl.shape[1]))), mode="edge")[:8 * rows, :8 * cols]
            blk = (p - 128).reshape(rows, 8, cols, 8).transpose(0, 2, 1, 3)
            d = dctn(blk, axes=(2, 3), norm="ortho").reshape(rows, cols, 64)
            self.coef.append(np.rint(d / np.asarray(self.q[self.comps[c][3]], np.float64)).astype(np.int64))

    def units(self, comps):
        """The blocks of a scan of components `comps` (indices), per unit in scan order: [[(c, by, bx), ...], ...]"""
        if len(comps) > 1:
            out = []
            for my in range(self.mcuy):
                for mx in range(self.mcux):
                    u = []
                    for c in comps:
                        _, ch, cv, _ = self.comps[c]
                        u += [(c, my * cv + v, mx * ch + hh) for v in range(cv) for hh in range(ch)]
                    out.append(u)
            return out
        c = comps[0]
        return [[(c, by, bx)] for by in range(-(-self.dh[c] // 8)) for bx in range(-(-self.dw[c] // 8))]


MAX_CORR_BITS = 1000                      # jcphuff.c: correction bits buffered before an EOB run is emitted


def scan_events(cf, comps, ss, se, ah, al, restart, eob_past_end=False, stats=None):
    """The events of one scan, one list per restart interval: ("h", table key, symbol) and ("b", bits, n).  The four scan kinds
    follow libjpeg's jcphuff.c (encode_mcu_DC_first / _DC_refine / _AC_first / _AC_refine); stats["zrl_refine"] counts the ZRL
    symbols of AC refinement scans."""
    out, units = [], cf.units(comps)
    step = restart or len(units)
    for i0 in range(0, len(units), step):
        ev, pred, st = [], {}, {"eobrun": 0, "be": []}

        def flush_eob(last=False):
            if st["eobrun"]:
                run = 0x7FFF if (last and eob_past_end) else st["eobrun"]
                nb = run.bit_length() - 1
                ev.append(("h", "ac", nb << 4))
                if nb:
                    ev.append(("b", run & ((1 << nb) - 1), nb))
                st["eobrun"] = 0
            ev.extend(("b", bit, 1) for bit in st["be"])        # the correction bits of the blocks in the run
            st["be"] = []

        for u in units[i0:i0 + step]:
            for c, by, bx in u:
                blk = cf.coef[c][by, bx]
                if ss == 0 and ah:
                    ev.append(("b", (int(blk[0]) >> al) & 1, 1))
                elif ss == 0:
                    v = int(blk[0]) >> al
                    d = v - pred.get(c, 0)
                    pred[c] = v
                    s = size(d)
                    ev.append(("h", "dc%d" % comps.index(c), s))
                    if s:
                        ev.append(("b", amplitude(d, s), s))
                elif ah == 0:
                    r = 0
                    for z in range(ss, se + 1):
                        x = int(blk[NATURAL[z]])
                        t = (abs(x) >> al) * (1 if x >= 0 else -1)
                        if t == 0:
                            r += 1
                            continue
                        flush_eob()
                        while r > 15:
                            ev.append(("h", "ac", 0xF0))
                            r -= 16
                        s = size(t)
                        ev.append(("h", "ac", r << 4 | s))
                        ev.append(("b", amplitude(t, s), s))
                        r = 0
                    if r:
                        st["eobrun"] += 1
                        if st["eobrun"] == 0x7FFF:
                            flush_eob()
                else:
                    absv = [abs(int(blk[NATURAL[z]])) >> al for z in range(64)]
                    eob = max([z for z in range(ss, se + 1) if absv[z] == 1], default=0)   # the last newly nonzero one
                    r, br = 0, []
                    for z in range(ss, se + 1):
                        t = absv[z]
                        if t == 0:
                            r += 1
                            continue
                        while r > 15 and z <= eob:
                            flush_eob()
                            ev.append(("h", "ac", 0xF0))
                            r -= 16
                            ev.extend(("b", bit, 1) for bit in br)
                            br = []
                            if stats is not None:
                                stats["zrl_refine"] = stats.get("zrl_refine", 0) + 1
                        if t > 1:                                    # already nonzero: a correction bit
                            br.append(t & 1)
                            continue
                        flush_eob()
                        ev.append(("h", "ac", r << 4 | 1))
                        ev.append(("b", 0 if blk[NATURAL[z]] < 0 else 1, 1))
                        ev.extend(("b", bit, 1) for bit in br)
                        br, r = [], 0
                    if r or br:
                        st["eobrun"] += 1
                        st["be"] += br
                        if st["eobrun"] == 0x7FFF or len(st["be"]) > MAX_CORR_BITS - 64 + 1:
                            flush_eob()
        flush_eob(last=True)
        out.append(ev)
    return out


def encode_progressive(cf, script, restart=0, dri=None, eob_past_end=(), extra=(), stats=None, app0=True):
    """A progressive file of coefficients cf: script [(comps, ss, se, ah, al)], a DHT (slots 0..) before every scan that needs
    one; dri {scan index: interval} writes a DRI before that scan (restart: the interval before the first); extra {scan index:
    [(marker, payload)]} more segments before a scan."""
    dri = dict(dri or {})
    hdr = [(0xE0, app0 if isinstance(app0, bytes) else b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0", b"")]
    for tq, q in sorted(cf.q.items()):
        hdr.append((0xDB, bytes([tq]) + bytes(q[NATURAL[k]] for k in range(64)), b""))
    sof = struct.pack(">BHHB", 8, cf.h, cf.w, len(cf.comps)) + b"".join(bytes([i, h << 4 | v, t]) for i, h, v, t in cf.comps)
    hdr.append((0xC2, sof, b""))
    ps, rst = hdr, restart
    if restart:
        ps.append((0xDD, struct.pack(">H", restart), b""))
    for si, (comps, ss, se, ah, al) in enumerate(script):
        ps += [(m, p, b"") for m, p in dict(extra).get(si, [])]
        if si in dri:
            rst = dri[si]
            ps.append((0xDD, struct.pack(">H", rst), b""))
        intervals = scan_events(cf, comps, ss, se, ah, al, rst, si in eob_past_end, stats)
        syms = {}
        for ev in intervals:
            for e in ev:
                if e[0] == "h":
                    syms.setdefault(e[1], []).append(e[2])
        tabs = {k: optimal(v) for k, v in sorted(syms.items())}
        dht = b"".join(t.dht(k == "ac", 0 if k == "ac" else int(k[2:])) for k, t in tabs.items())
        if dht:
            ps.append((0xC4, dht, b""))
        pieces = []
        for ev in intervals:
            b = Bits()
            for e in ev:
                if e[0] == "h":
                    code, ln = tabs[e[1]].code[e[2]]
                    b.put(code, ln)
                elif e[2]:
                    b.put(e[1], e[2])
            pieces.append(b.flush())
        data = pieces[0] + b"".join(bytes([0xFF, 0xD0 + (k & 7)]) + p for k, p in enumerate(pieces[1:]))
        ids = [(cf.comps[c][0], comps.index(c) if (ss == 0 and not ah) else 0, 0) for c in comps]
        ps.append((0xDA, sos(ids, ss, se, ah, al), data))
    return build(ps)


def bands(rs, lo, hi, ncut, narrow=False):
    """A random partition of lo..hi into bands [(a, b)]: ncut random cuts, and a 1-wide band somewhere when narrow"""
    cuts = set(int(x) for x in rs.randint(lo + 1, hi + 1, ncut)) if hi > lo else set()
    if narrow and hi > lo:
        k = int(rs.randint(lo, hi + 1))
        cuts |= {x for x in (k, k + 1) if lo < x <= hi}
    edges = [lo] + sorted(cuts) + [hi + 1]
    return [(a, b - 1) for a, b in zip(edges, edges[1:])]


def random_script(rs, ncomp, max_al=13, wide=False, ac_chains=False):
    """A complete script: DC first (interleaved over all, 2 + 1 or one per component) at a random Al with its refinement chain,
    then each component's bands 1..63 (1-wide, and the DC chain from max_al, when wide) as AC first scans, in a random order
    keeping each chain in order.  Without ac_chains the AC scans are at Al 0.  With it each component's AC coefficients start at
    a random Al (up to 13) and are refined down to 0 one bit plane at a time, each plane cut into its own random bands (narrow
    and 1-wide ones among them, bands starting after 1 and ending before 63)."""
    mode = rs.randint(3) if ncomp == 3 else 2
    groups = [[0, 1, 2]] if mode == 0 else ([[0, 1], [2]] if mode == 1 else [[c] for c in range(ncomp)])
    first, later = [], []
    for g in groups:
        al = max_al if wide else int(rs.randint(0, max_al + 1))
        first.append((g, 0, 0, 0, al))
        later.append([(g, 0, 0, a + 1, a) for a in range(al - 1, -1, -1)])
    for c in range(ncomp):
        if ac_chains:
            top = int(rs.choice([0, 1, 2, 3, 5, 13]))
            chain = []
            for a in range(top, -1, -1):
                ah = 0 if a == top else a + 1
                chain += [([c], lo, hi, ah, a) for lo, hi in bands(rs, 1, 63, int(rs.randint(0, 3 if top > 5 else 6)), rs.rand() < 0.5)]
            later.append(chain)
            continue
        if wide:
            cuts = list(range(2, 64))
        else:
            cuts = sorted(set(int(x) for x in rs.randint(2, 64, rs.randint(2, 9))) | {63})
        lo, bs = 1, []
        for cut in cuts + [64]:
            if cut > lo:
                bs.append(([c], lo, cut - 1, 0, 0))
                lo = cut
        later.append(bs)
    script = list(first)
    while any(later):
        ch = [i for i, l in enumerate(later) if l]
        script.append(later[ch[rs.randint(len(ch))]].pop(0))
    return script


def ac_script(rs, ncomp):
    """random_script with AC approximation chains, drawn again until it fits the decoder's 128 scans"""
    while True:
        s = random_script(rs, ncomp, ac_chains=True)
        if len(s) <= 128:
            return s


# ---- families -------------------------------------------------------------------------------------------------------------------
def cv2_prog(cv2, img, q=90, sampling=None, rst=0, progressive=1):
    params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, progressive, cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if sampling:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + sampling)]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def cv2_files(cv2):
    import jpeg_cases as jc
    from make_golden_jpeg import exif_app1
    out, seed = {}, 4000

    def enc(name, seed, h, w, s, q=90, rst=0):
        img = jc.image(seed, h, w, smooth=(h * w > 1_000_000))
        if s == "grey":
            out[name] = cv2_prog(cv2, cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), q, None, rst)
        else:
            out[name] = cv2_prog(cv2, img, q, s, rst)

    for s in jc.SAMPLINGS:
        for q in (1, 50, 95, 100):
            seed += 1
            enc("cv2_q%d_%s" % (q, s), seed, 37, 53, s, q)
        for (h, w) in ((1, 1), (1, 17), (17, 1), (8, 8), (15, 9), (16, 16), (31, 33), (37, 53), (333, 500)):
            seed += 1
            enc("cv2_size%dx%d_%s" % (h, w, s), seed, h, w, s)
        for r in (1, 7):
            seed += 1
            enc("cv2_rst%d_%s" % (r, s), seed, 45, 70, s, 90, r)
    for o in (6, 8):
        for order in ("II", "MM"):
            seed += 1
            b = cv2_prog(cv2, jc.image(seed, 37, 53), 90, "420" if order == "II" else "422")
            out["cv2_exif%d_%s" % (o, order)] = b[:2] + exif_app1(o, order) + b[2:]
    enc("cv2_fullhd_420", 2001, 1080, 1920, "420")
    return out


def pillow_files():
    from PIL import Image
    import jpeg_cases as jc
    out = {}

    def save(name, img, **kw):
        b = io.BytesIO()
        img.save(b, "JPEG", progressive=True, **kw)
        out[name] = b.getvalue()

    rgb = Image.fromarray(jc.image(5001, 45, 70)[..., ::-1].copy())
    for s in (0, 1, 2):
        for q in (5, 50, 95):
            save("pil_sub%d_q%d" % (s, q), rgb, quality=q, subsampling=s)
    save("pil_optimize", rgb, quality=80, optimize=True)
    save("pil_grey", rgb.convert("L"), quality=80)
    return out


# libjpeg's jpeg_simple_progression for YCbCr, which cv2 and Pillow write
CV2_SCRIPT = [([0, 1, 2], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([2], 1, 63, 0, 1), ([1], 1, 63, 0, 1), ([0], 6, 63, 0, 2),
              ([0], 1, 63, 2, 1), ([0, 1, 2], 0, 0, 1, 0), ([2], 1, 63, 1, 0), ([1], 1, 63, 1, 0), ([0], 1, 63, 1, 0)]


def baseline_coefs(b):
    """A Coefs holding the quantised coefficients of a baseline file (8-bit DQT, one interleaved Huffman scan, no restart
    markers), read by a small decoder: what a lossless re-code to progressive keeps."""
    cf = Coefs.__new__(Coefs)
    q, dc, ac, pos = {}, {}, {}, 2
    while True:
        m, n = b[pos + 1], struct.unpack(">H", b[pos + 2:pos + 4])[0]
        p, pos = b[pos + 4:pos + 2 + n], pos + 2 + n
        if m == 0xDB:
            for o in range(0, len(p), 65):
                assert p[o] >> 4 == 0
                q[p[o] & 15] = [0] * 64
                for k in range(64):
                    q[p[o] & 15][NATURAL[k]] = p[o + 1 + k]
        elif m == 0xC4:
            o = 0
            while o < len(p):
                cnt, vals = p[o + 1:o + 17], p[o + 17:o + 17 + sum(p[o + 1:o + 17])]
                codes, code, i = {}, 0, 0
                for ln in range(1, 17):
                    for _ in range(cnt[ln - 1]):
                        codes[(ln, code)] = vals[i]
                        code, i = code + 1, i + 1
                    code <<= 1
                (ac if p[o] >> 4 else dc)[p[o] & 15] = codes
                o += 17 + len(vals)
        elif m == 0xC0:
            cf.h, cf.w = struct.unpack(">HH", p[1:5])
            cf.comps = [(p[6 + 3 * c], p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15, p[8 + 3 * c]) for c in range(p[5])]
        elif m == 0xDD:
            assert struct.unpack(">H", p)[0] == 0
        elif m == 0xDA:
            sel = [(p[2 + 2 * k] >> 4, p[2 + 2 * k] & 15) for k in range(p[0])]
            break
    cf.q = q
    cf.hmax, cf.vmax = max(c[1] for c in cf.comps), max(c[2] for c in cf.comps)
    cf.mcux, cf.mcuy = -(-cf.w // (8 * cf.hmax)), -(-cf.h // (8 * cf.vmax))
    cf.dw = [-(-cf.w * c[1] // cf.hmax) for c in cf.comps]
    cf.dh = [-(-cf.h * c[2] // cf.vmax) for c in cf.comps]
    cf.coef = [np.zeros((cf.mcuy * c[2], cf.mcux * c[1], 64), np.int64) for c in cf.comps]
    data = b[pos:b.rindex(b"\xff\xd9")].replace(b"\xff\x00", b"\xff")
    bits = np.unpackbits(np.frombuffer(data, np.uint8)).tolist()
    at = [0]

    def get(n):
        v = 0
        for _ in range(n):
            v = v << 1 | bits[at[0]]
            at[0] += 1
        return v

    def sym(t):
        code = 0
        for ln in range(1, 17):
            code = code << 1 | get(1)
            if (ln, code) in t:
                return t[(ln, code)]
        raise ValueError("bad code")

    def extend(v, s):
        return v - (1 << s) + 1 if v < (1 << (s - 1)) else v

    pred = [0] * len(cf.comps)
    for u in cf.units(list(range(len(cf.comps)))):
        for c, by, bx in u:
            blk = cf.coef[c][by, bx]
            s = sym(dc[sel[c][0]])
            pred[c] += extend(get(s), s) if s else 0
            blk[0] = pred[c]
            k = 1
            while k < 64:
                rs = sym(ac[sel[c][1]])
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    blk[NATURAL[k]] = extend(get(s), s)
                    k += 1
                elif r == 15:
                    k += 16
                else:
                    break
    return cf


def tx_files():
    """The reference's photos re-coded losslessly as progressive files: their coefficients, tables and geometry kept, scanned by
    cv2's script and by a seeded other one (AC approximation chains included)"""
    out = {}
    for k, stem in enumerate(PHOTOS):
        with open(os.path.join(HERE, stem + ".jpg"), "rb") as f:
            cf = baseline_coefs(f.read())
        out["tx_cv2_" + stem] = encode_progressive(cf, CV2_SCRIPT)
        out["tx_seeded_" + stem] = encode_progressive(cf, ac_script(np.random.RandomState(7500 + k), 3))
    return out


def coef_sets():
    import jpeg_cases as jc
    return {"420": Coefs(jc.image(6001, 37, 53), (2, 2), [[max(1, v // 4) for v in SCALE], [max(1, v // 3) for v in SCALE]]),
            "444": Coefs(jc.image(6002, 31, 33), (1, 1), [[1] * 64, [1] * 64]),
            "grey": Coefs(jc.image(6003, 37, 53), (1, 1), [[max(1, v // 5) for v in SCALE]], grey=True)}


def script_files():
    out, sets = {}, coef_sets()
    for name, cf in sets.items():
        nc = len(cf.comps)
        for k in range(6):
            rs = np.random.RandomState(7000 + 10 * k + nc)
            out["script_%s_%d" % (name, k)] = encode_progressive(cf, random_script(rs, nc), restart=int(rs.choice([0, 0, 2, 5])))
        # a DC chain from Al 13 to 0 and 1-wide bands over every coefficient: 14 + 63 scans of one component
        if nc == 1:
            out["script_grey_wide"] = encode_progressive(cf, random_script(np.random.RandomState(7100), 1, wide=True))
        # AC approximation chains: AC refinement scans over random, narrow and 1-wide bands, from Al up to 13
        for k in range(6):
            rs = np.random.RandomState(7300 + 10 * k + nc)
            out["script_ac_%s_%d" % (name, k)] = encode_progressive(cf, ac_script(rs, nc), restart=int(rs.choice([0, 0, 3, 7])))
        # the baseline coefficients of the set, one scan per coefficient group: what every script above must decode to
        out["script_%s_flat" % name] = encode_progressive(cf, [(list(range(nc)), 0, 0, 0, 0)] + [([c], 1, 63, 0, 0) for c in range(nc)])
    return out, sets


def enc_files(sets):
    import jpeg_cases as jc
    out = {}
    cf, nc = sets["420"], 3
    script = random_script(np.random.RandomState(7200), nc)
    out["enc_dri_between_scans"] = encode_progressive(cf, script, restart=3, dri={2: 0, 4: 5, 6: 1, 9: 4})
    out["enc_rst_not_row"] = encode_progressive(cf, script, restart=3)
    out["enc_eob_past_segment"] = encode_progressive(cf, script, restart=4, eob_past_end=set(range(len(script))))
    big = Coefs(jc.image(6004, 1088, 1024, smooth=True), (1, 1), [[max(1, v // 2) for v in SCALE]], grey=True)
    out["enc_eob14_rows"] = encode_progressive(big, [([0], 0, 0, 0, 0), ([0], 1, 2, 0, 0), ([0], 3, 40, 0, 0), ([0], 41, 63, 0, 0)])
    ext = Coefs(jc.image(6005, 16, 16), (1, 1), [[1] * 64], grey=True)
    ext.coef[0][..., 0] = np.array([[-2047, 2047], [1023, -1024]])
    out["enc_dc_al13"] = encode_progressive(ext, [([0], 0, 0, 0, 13)] + [([0], 0, 0, a + 1, a) for a in range(12, -1, -1)] +
                                            [([0], 1, 63, 0, 0)])
    # AC at Al 13: extreme coefficients (16 bits of magnitude) sent 13 bit planes down, then refined one plane at a time over
    # bands that start after 1 and end before 63
    big_ac = Coefs(jc.image(6006, 16, 16), (1, 1), [[1] * 64], grey=True)
    for z, v in ((1, 32767), (2, -32767), (9, 16384), (20, -8193), (40, 8191), (63, -24576)):
        big_ac.coef[0][0, 0, NATURAL[z]] = v
        big_ac.coef[0][1, 1, NATURAL[z]] = -v
    chain = [([0], 0, 0, 0, 0), ([0], 1, 63, 0, 13)]
    for a in range(12, -1, -1):
        chain += [([0], 1, 1, a + 1, a), ([0], 2, 39, a + 1, a), ([0], 40, 62, a + 1, a), ([0], 63, 63, a + 1, a)]
    out["enc_ac_al13"] = encode_progressive(big_ac, chain)
    # ZRL in AC refinement: 16 or more zero-history coefficients before a newly nonzero one
    stats = {}
    out["enc_zrl_refine"] = encode_progressive(sets["grey"], [([0], 0, 0, 0, 0), ([0], 1, 63, 0, 1), ([0], 1, 63, 1, 0)],
                                               stats=stats)
    assert stats.get("zrl_refine", 0) > 0
    return out


def rewritten_files(cv2):
    """cv2 progressive files with scans rewritten (accepted), refused scripts and damaged scans"""
    import jpeg_cases as jc
    base = cv2_prog(cv2, jc.image(8001, 37, 53), 90, "420")
    ps = parts(base)
    si = scan_indices(ps)
    assert len(si) == 10
    out = {"enc_base": base}
    # a DQT redefining table 0 after scan 0 (which latched it for Y) and table 1 after scan 2 (Cr's first AC scan; Cb and Cr
    # latched it at scan 0): the decode keeps the latched tables
    dq = lambda t: (0xDB, bytes([t]) + bytes([99] * 64), b"")  # noqa: E731
    out["enc_dqt_after_first_scan"] = build(ps[:si[1]] + [dq(0)] + ps[si[1]:si[3]] + [dq(1)] + ps[si[3]:])
    # the DC refinement (scan 6) naming tables 3, which are never defined
    m, p, d = ps[si[6]]
    assert p[0] == 3 and p[-1] >> 4 == 1
    out["enc_dc_refine_undefined_tables"] = build(ps[:si[6]] + [(m, bytes([3, p[1], 0x33, p[3], 0x33, p[5], 0x33]) + p[7:], d)] +
                                                  ps[si[6] + 1:])
    # every size-1 symbol of the AC refinement scans' tables (scans 5, 7, 8, 9) given size 2: libjpeg-turbo reads one bit anyway
    q = list(ps)
    for k in (5, 7, 8, 9):
        i = si[k] - 1
        assert q[i][0] == 0xC4
        m, p, d = q[i]
        nvals = sum(p[1:17])
        vals = bytes(v + 1 if v & 15 == 1 else v for v in p[17:17 + nvals])
        q[i] = (m, p[:17] + vals + p[17 + nvals:], d)
    out["enc_refine_size2"] = build(q)
    # refused: the trailing scans dropped, EOI kept
    for k in range(1, 10):
        out["bad_first_%d_scans" % k] = build(ps[:si[k]])
    grey = parts(cv2_prog(cv2, cv2.cvtColor(jc.image(8002, 37, 53), cv2.COLOR_BGR2GRAY), 90))
    g = [i for i, x in enumerate(grey) if x[0] == 0xC2][0]
    sof = grey[g][1]
    grey[g] = (0xC2, sof[:5] + bytes([3]) + sof[6:9] + bytes([2, 0x11, 0, 3, 0x11, 0]), b"")
    out["bad_component_never_scanned"] = build(grey)
    out["bad_dc_se1"] = build(with_sos(ps, 0, se=1))
    out["bad_ac_ss_after_se"] = build(with_sos(ps, 1, ss=6, se=5))
    out["bad_ac_se64"] = build(with_sos(ps, 1, se=64))
    m, p, d = ps[si[1]]
    out["bad_ac_two_components"] = build(ps[:si[1]] + [(m, bytes([2]) + p[1:3] + bytes([2, 0x11]) + p[3:], d)] + ps[si[1] + 1:])
    out["bad_ah_al"] = build(with_sos(ps, 5, ah=2, al=0))
    out["bad_al14"] = build(with_sos(ps, 0, al=14))
    out["bogus_ac_before_dc"] = build(ps[:si[0] - 1] + ps[si[1] - 1:si[1] + 1] + ps[si[0] - 1:si[0] + 1] + ps[si[1] + 1:])
    out["bogus_ah"] = build(with_sos(ps, 5, ah=3, al=2))
    m, p, d = ps[si[0]]
    out["bad_dc_components_out_of_order"] = build(ps[:si[0]] + [(m, p[:1] + p[3:5] + p[1:3] + p[5:], d)] + ps[si[0] + 1:])
    out["bad_sof10"] = base.replace(b"\xff\xc2", b"\xff\xca", 1)
    # damaged
    s9 = si[9]
    pre = len(build(ps[:s9], eoi=False)) + 4 + len(ps[s9][1])                # offset of scan 9's data
    s0 = len(build(ps[:si[0]], eoi=False)) + 4 + len(ps[si[0]][1])
    out["cut_first_scan"] = base[:s0 + len(ps[si[0]][2]) // 2]
    out["cut_refinement"] = base[:pre + len(ps[s9][2]) // 2]
    out["cut_between_scans"] = build(ps[:si[5]], eoi=False)
    out["cut_before_eoi"] = base[:-2]
    out["cut_eoi_d9"] = base[:-1]
    for k in range(3):
        rs = np.random.RandomState(8100 + k)
        b = bytearray(base)
        data = ps[s9][2]
        for _ in range(3):
            while True:
                o = int(rs.randint(len(data) - 2))
                if data[o] != 0xFF and data[o - 1] != 0xFF and data[o + 1] != 0x00:
                    break
            b[pre + o] = int(rs.randint(0, 255))
        out["corrupt_refinement_%d" % k] = bytes(b)
    # an AC refinement symbol whose zero run carries it past its band (1..5): libjpeg writes coefficient 6 (complete since a
    # level-0 scan); the scan is alone on its level, so the decode writes it after that scan too
    cf = Coefs(jc.image(8004, 16, 16), (1, 1), [[2] * 64], grey=True)
    for z in range(1, 6):
        cf.coef[0][..., NATURAL[z]] = 0
    head = parts(encode_progressive(cf, [([0], 0, 0, 0, 0), ([0], 1, 5, 0, 1), ([0], 6, 63, 0, 0)]))
    t = Table([(0xA1, 1), (0x10, 2)])
    bb = Bits()
    for code, n in ((0, 1), (1, 1), (0b10, 2), (1, 1)):               # block 0: run 10 then +1; blocks 1-3: EOB run of 3
        bb.put(code, n)
    out["corrupt_run_past_band"] = build(head + [(0xC4, t.dht(1, 0), b""), (0xDA, sos([(1, 0, 0)], 1, 5, 1, 0), bb.flush())])
    rb = cv2_prog(cv2, jc.image(8003, 37, 53), 90, "420", rst=2)
    rp = parts(rb)
    ri = scan_indices(rp)
    m, p, d = rp[ri[7]]
    k = d.index(b"\xff\xd2")
    out["rst_renumbered_in_refinement"] = build(rp[:ri[7]] + [(m, p, d[:k + 1] + b"\xd3" + d[k + 2:])] + rp[ri[7] + 1:])
    return out


def too_many_scans(sets):
    """All 1-wide bands of the three components: more scans than the decoder takes"""
    cf = sets["420"]
    script = [([0, 1, 2], 0, 0, 0, 0)] + [([c], k, k, 0, 0) for c in range(3) for k in range(1, 64)]
    return {"bad_too_many_scans": encode_progressive(cf, script)}


def main():
    import cv2
    import PIL
    import jpeg_cases as jc
    import jpeg_progressive_cases as pc
    files = {}
    files.update(cv2_files(cv2))
    files.update(pillow_files())
    files.update(tx_files())
    sc, sets = script_files()
    files.update(sc)
    files.update(enc_files(sets))
    files.update(rewritten_files(cv2))
    files.update(too_many_scans(sets))
    assert sorted(files) == sorted(pc.CASES), sorted(set(files) ^ set(pc.CASES))
    out, dec = {}, {}
    for name in pc.CASES:
        buf = np.frombuffer(files[name], np.uint8)
        out["jpg_" + name] = buf
        d = dec[name] = cv2.imdecode(buf, cv2.IMREAD_COLOR)
        if d is None:
            out["none_" + name] = np.ones(1, np.uint8)
            continue
        out["shape_" + name] = np.array(d.shape, np.int64)
        out["sha_" + name] = jc.digest(d)
        if d.nbytes <= jc.FULL_BYTES:
            out["bgr_" + name] = d
    # what the families rest on
    modelzoo = np.load(os.path.join(HERE, "frames_modelzoo.npz"))
    for stem in PHOTOS:
        for kind in ("cv2", "seeded"):
            assert np.array_equal(dec["tx_%s_%s" % (kind, stem)], modelzoo[stem]), (kind, stem)
    for s in ("420", "444", "grey"):
        for name in pc.CASES:
            if name.startswith(("script_%s_" % s, "script_ac_%s_" % s)):
                assert np.array_equal(dec[name], dec["script_%s_flat" % s]), name
    assert np.array_equal(dec["script_grey_wide"], dec["script_grey_flat"])
    for name in ("enc_dqt_after_first_scan", "enc_dc_refine_undefined_tables", "enc_refine_size2"):
        assert np.array_equal(dec[name], dec["enc_base"]), name
    for name in ("bad_dc_se1", "bad_ac_ss_after_se", "bad_ac_se64", "bad_ac_two_components", "bad_ah_al", "bad_al14"):
        assert dec[name] is None, name
    for name in pc.CASES:
        if name.startswith("cut_"):
            assert dec[name] is None, name
    np.savez_compressed(os.path.join(HERE, "jpeg_progressive.npz"), **out)
    meta = {"generator": "tests/golden/make_golden_jpeg_progressive.py", "opencv": cv2.__version__, "pillow": PIL.__version__,
            "libjpeg_turbo": "3.1.2 (OpenCV's bundled build-libjpeg-turbo, x86-64 SIMD)", "numpy": np.__version__,
            "cases": len(pc.CASES), "cv2_none": sorted(n for n in pc.CASES if "none_" + n in out)}
    with open(os.path.join(HERE, "META_jpeg_progressive.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    print("wrote %d cases (%d that cv2 cannot decode), %d bytes" % (
        len(pc.CASES), len(meta["cv2_none"]), os.path.getsize(os.path.join(HERE, "jpeg_progressive.npz"))))


if __name__ == "__main__":
    main()
