"""A baseline / extended sequential Huffman JPEG writer (ITU T.81) for the decoder tests, in pure Python and numpy.

It takes quantised coefficients per block, not pixels, so a test can put any value at any zigzag position, and it
controls the stream around them: 8- or 16-bit quantisation tables with SOF0 or SOF1, Huffman tables given as a
counts / symbols pair or built from symbol frequencies (T.81 Annex K.2, lengths limited to 16) in slots 0-3, shared
or separate per component, component ids, sampling factors, DRI and the restart segments, JFIF (APP0) and Adobe
(APP14) segments, and the marker order (tables after SOF, tables redefined before SOS).

    blob = write(width, height, comps, blocks, quant, dc, ac, ...)

comps: one dict per component: id, h, v, tq (quantisation slot), td / ta (DC / AC Huffman slots).
blocks: per component an int array [rows, cols, 64] of quantised coefficients in zigzag order over the component's
block grid (rows = mcuy * v, cols = mcux * h, padding blocks included).  Index 0 holds the DC *value* as an
unbounded integer; the writer codes the differences (reset at each restart), so a run of DC values can leave int16
while every difference stays in category 11.
quant: {slot: 64 values in zigzag order}; dc, ac: {slot: (counts, symbols)}."""
import numpy as np

# zigzag index -> natural (row-major) position
NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                    13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                    45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)


def category(v):
    """the magnitude category (SSSS) of a coefficient value"""
    return int(abs(int(v))).bit_length()


def huff_from_freqs(freq, limit=16):
    """(counts, symbols) of a Huffman table for symbol frequencies freq[0..255] (zero: symbol absent), built as T.81
    Annex K.2 does: code sizes with a reserved all-ones code point, then lengths above `limit` folded down (K.3),
    symbols ordered by code length, then by value."""
    f = [int(x) for x in freq] + [1]                      # symbol 256: the reserved code point
    size = [0] * 257
    others = [-1] * 257
    while True:
        live = [i for i in range(257) if f[i] > 0]
        if len(live) < 2:
            break
        v1 = min(live, key=lambda i: (f[i], -i))
        v2 = min((i for i in live if i != v1), key=lambda i: (f[i], -i))
        f[v1] += f[v2]
        f[v2] = 0
        size[v1] += 1
        while others[v1] >= 0:
            v1 = others[v1]
            size[v1] += 1
        others[v1] = v2
        size[v2] += 1
        while others[v2] >= 0:
            v2 = others[v2]
            size[v2] += 1
    bits = [0] * 33
    for s in size:
        if s:
            bits[s] += 1
    for i in range(32, limit, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = limit
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                           # drop the reserved code point
    syms = [s for ln in range(1, 33) for s in range(256) if size[s] == ln]
    return bytes(bits[1:17]), bytes(syms)


def codes(counts, syms):
    """{symbol: (code, length)} of the canonical code of a (counts, symbols) table"""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out[syms[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return out


class _Bits:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def put(self, code, ln):
        self.acc = (self.acc << ln) | (code & ((1 << ln) - 1))
        self.n += ln
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 0xFF
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)                         # byte stuffing
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)  # pad with one bits


def block_symbols(zz):
    """the (symbol, extra bits value, size) sequence of a block's AC coefficients (zigzag 1..63) as an encoder writes
    it: (run, size) symbols, ZRL for each 16 zeros before a nonzero value, EOB unless coefficient 63 is nonzero"""
    out, run = [], 0
    for k in range(1, 64):
        v = int(zz[k])
        if v == 0:
            run += 1
            continue
        while run > 15:
            out.append((0xF0, 0, 0))
            run -= 16
        s = category(v)
        out.append(((run << 4) | s, v, s))
        run = 0
    if run:
        out.append((0x00, 0, 0))
    return out


def _extra(v, s):
    return v if v >= 0 else v + (1 << s) - 1


def _seg(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def dqt(slot, q, sixteen=False):
    q = [int(x) for x in q]
    if sixteen:
        return _seg(0xDB, bytes([0x10 | slot]) + b"".join(x.to_bytes(2, "big") for x in q))
    return _seg(0xDB, bytes([slot] + q))


def dht(tc, slot, table):
    counts, syms = table
    return _seg(0xC4, bytes([(tc << 4) | slot]) + bytes(counts) + bytes(syms))


def jfif():
    return _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")


def adobe(transform):
    return _seg(0xEE, b"Adobe\0\x64\0\0\0\0" + bytes([transform]))


def mcu_shape(width, height, comps):
    """(mcux, mcuy) of a frame; one component: one block per MCU, as for a non-interleaved scan"""
    if len(comps) == 1:
        return -(-width // 8), -(-height // 8)
    hmax, vmax = max(c["h"] for c in comps), max(c["v"] for c in comps)
    return -(-width // (8 * hmax)), -(-height // (8 * vmax))


def block_grid(width, height, comps, ci):
    """(rows, cols) of component ci's block grid, padding blocks included"""
    mcux, mcuy = mcu_shape(width, height, comps)
    if len(comps) == 1:
        return mcuy, mcux
    return mcuy * comps[ci]["v"], mcux * comps[ci]["h"]


def scan(width, height, comps, blocks, dc, ac, restart=0, ac_symbols=None):
    """the entropy-coded data with its RSTn markers.  ac_symbols: {(component, row, col): [(symbol, value), ...]}
    replaces a block's AC symbols as written (for EOB / ZRL sequences no encoder emits)."""
    tabs = [(codes(*dc[c["td"]]), codes(*ac[c["ta"]])) for c in comps]
    out, bw = bytearray(), _Bits()
    prev = [0] * len(comps)
    last = -1
    for m, ci, r, col in walk(width, height, comps):
        if m != last and restart and m and m % restart == 0:
            bw.flush()
            out += bw.out + bytes([0xFF, 0xD0 + (m // restart - 1) % 8])
            bw = _Bits()
            prev = [0] * len(comps)
        last = m
        dct, act = tabs[ci]
        zz = blocks[ci][r, col]
        diff = int(zz[0]) - prev[ci]
        prev[ci] = int(zz[0])
        s = category(diff)
        bw.put(*dct[s])
        if s:
            bw.put(_extra(diff, s), s)
        syms = ac_symbols.get((ci, r, col)) if ac_symbols else None
        if syms is None:
            syms = [(sym, v) for sym, v, _ in block_symbols(zz)]
        for sym, v in syms:
            bw.put(*act[sym])
            if sym & 15:
                bw.put(_extra(v, sym & 15), sym & 15)
    bw.flush()
    return bytes(out + bw.out)


def write(width, height, comps, blocks, quant, dc, ac, restart=0, sixteen=False, sof1=False, app=("jfif",),
          order=("dqt", "sof", "dht", "dri"), decoys=(), ac_symbols=None, exif=None):
    """a whole stream: SOI, the APPn segments of `app` ("jfif", ("adobe", transform)), the table / frame segments in
    `order`, then SOS, the scan and EOI.  decoys: segments written first that the real tables later redefine (the
    last definition wins).  sixteen: 16-bit quantisation tables (needs SOF1 for a standard stream; sof1 picks it)."""
    parts = [b"\xff\xd8"]
    for a in app:
        parts.append(jfif() if a == "jfif" else adobe(a[1]))
    parts += list(decoys)
    sof = bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([len(comps)])
    for c in comps:
        sof += bytes([c["id"], (c["h"] << 4) | c["v"], c["tq"]])
    segs = {"dqt": b"".join(dqt(s, q, sixteen) for s, q in sorted(quant.items())),
            "sof": _seg(0xC1 if sof1 else 0xC0, sof),
            "dht": b"".join(dht(0, s, t) for s, t in sorted(dc.items())) + b"".join(
                dht(1, s, t) for s, t in sorted(ac.items())),
            "dri": _seg(0xDD, restart.to_bytes(2, "big")) if restart else b""}
    parts += [segs[k] for k in order]
    sos = bytes([len(comps)]) + b"".join(bytes([c["id"], (c["td"] << 4) | c["ta"]]) for c in comps) + b"\x00\x3f\x00"
    parts.append(_seg(0xDA, sos))
    parts.append(scan(width, height, comps, blocks, dc, ac, restart, ac_symbols))
    parts.append(b"\xff\xd9")
    blob = b"".join(parts)
    if exif is not None:
        from jpeg_cases import with_orientation
        blob = with_orientation(blob, exif)
    return blob


def walk(width, height, comps):
    """the blocks in decode order: (mcu, component, row, col), MCU by MCU, component by component"""
    mcux, mcuy = mcu_shape(width, height, comps)
    one = len(comps) == 1
    for m in range(mcux * mcuy):
        my, mx = divmod(m, mcux)
        for ci, c in enumerate(comps):
            hh, vv = (1, 1) if one else (c["h"], c["v"])
            for by in range(vv):
                for bx in range(hh):
                    yield m, ci, my * vv + by, mx * hh + bx


def optimal_tables(width, height, comps, blocks, restart=0, limit=16):
    """(comps, dc, ac): tables built from the symbol frequencies of the blocks, one DC / AC pair per component in
    slots 0, 1, 2, and comps pointing at them"""
    fd = np.zeros((len(comps), 256), np.int64)
    fa = np.zeros((len(comps), 256), np.int64)
    prev = [0] * len(comps)
    last = -1
    for m, ci, r, col in walk(width, height, comps):
        if m != last and restart and m % restart == 0:
            prev = [0] * len(comps)
        last = m
        zz = blocks[ci][r, col]
        fd[ci, category(int(zz[0]) - prev[ci])] += 1
        prev[ci] = int(zz[0])
        for sym, _, _ in block_symbols(zz):
            fa[ci, sym] += 1
    dc = {ci: huff_from_freqs(fd[ci], limit) for ci in range(len(comps))}
    ac = {ci: huff_from_freqs(fa[ci], limit) for ci in range(len(comps))}
    return [dict(c, td=ci, ta=ci) for ci, c in enumerate(comps)], dc, ac


def read_cv2_stream(blob):
    """the frame, tables and quantised blocks of a baseline stream cv2 wrote, decoded with the decoder's own parser:
    (width, height, comps, blocks, quant, dc, ac, restart) in write()'s form, DC as values"""
    from rotate_yolov3_b200.decode import _NATURAL, parse
    d = np.frombuffer(blob, np.uint8)
    hd = parse(d)
    raw = _tables(d)
    comps, quant = [], {}
    for ci, (cid, h, v, tq, td, ta) in enumerate(raw["comps"]):
        comps.append({"id": cid, "h": h, "v": v, "tq": tq, "td": td, "ta": ta})
    for s, q in raw["quant"].items():
        quant[s] = q
    blocks = _entropy_decode(d, hd, comps, raw)
    return hd.width, hd.height, comps, blocks, quant, raw["dc"], raw["ac"], hd.restart


def _tables(d):
    i, n = 2, len(d)
    out = {"quant": {}, "dc": {}, "ac": {}, "comps": None}
    frame = None
    while i < n:
        while d[i] == 0xFF:
            i += 1
        m = int(d[i])
        ln = (int(d[i + 1]) << 8) | int(d[i + 2])
        seg = bytes(d[i + 3:i + 1 + ln])
        if m == 0xDB:
            k = 0
            while k < len(seg):
                pq, tq = seg[k] >> 4, seg[k] & 15
                if pq:
                    vals = [int.from_bytes(seg[k + 1 + 2 * j:k + 3 + 2 * j], "big") for j in range(64)]
                else:
                    vals = list(seg[k + 1:k + 65])
                out["quant"][tq] = vals
                k += 1 + (128 if pq else 64)
        elif m == 0xC4:
            k = 0
            while k < len(seg):
                tc, th = seg[k] >> 4, seg[k] & 15
                counts = seg[k + 1:k + 17]
                cnt = sum(counts)
                out["dc" if tc == 0 else "ac"][th] = (bytes(counts), bytes(seg[k + 17:k + 17 + cnt]))
                k += 17 + cnt
        elif m in (0xC0, 0xC1):
            frame = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(seg[5])]
        elif m == 0xDA:
            tabs = [(seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15) for c in range(seg[0])]
            out["comps"] = [f + t for f, t in zip(frame, tabs)]
            out["scan"] = i + 1 + ln
            return out
        i += 1 + ln
    raise ValueError("no scan")


def _entropy_decode(d, hd, comps, raw):
    """the quantised blocks of the scan (a plain serial decoder, for reading cv2's streams back)"""
    tabs = [({v: k for k, v in codes(*raw["dc"][c["td"]]).items()}, {v: k for k, v in codes(*raw["ac"][c["ta"]]).items()})
            for c in comps]
    starts, ends, first, nmcu = hd.segments
    one = len(comps) == 1
    blocks = [np.zeros(block_grid(hd.width, hd.height, comps, ci) + (64,), np.int64) for ci in range(len(comps))]
    for s, e, f0, nm in zip(starts, ends, first, nmcu):
        data = bytes(d[s:e]).replace(b"\xff\x00", b"\xff")
        bits = "".join(format(b, "08b") for b in data)
        p = 0
        prev = [0] * len(comps)

        def sym(tab):
            nonlocal p
            for ln in range(1, 17):
                k = (int(bits[p:p + ln], 2), ln)
                if k in tab:
                    p += ln
                    return tab[k]
            raise ValueError("bad code")

        def val(s):
            nonlocal p
            if s == 0:
                return 0
            r = int(bits[p:p + s], 2)
            p += s
            return r if r >= 1 << (s - 1) else r - (1 << s) + 1

        for m in range(int(f0), int(f0 + nm)):
            my, mx = divmod(m, hd.mcux)
            for ci, c in enumerate(comps):
                hh, vv = (1, 1) if one else (c["h"], c["v"])
                for by in range(vv):
                    for bx in range(hh):
                        zz = blocks[ci][my * vv + by, mx * hh + bx]
                        prev[ci] += val(sym(tabs[ci][0]))
                        zz[0] = prev[ci]
                        k = 1
                        while k < 64:
                            rs = sym(tabs[ci][1])
                            if rs == 0:
                                break
                            if rs == 0xF0:
                                k += 16
                                continue
                            k += rs >> 4
                            zz[k] = val(rs & 15)
                            k += 1
    return blocks
