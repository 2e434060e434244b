"""JPEG decoding on the device: the file contents in, what ``cv2.imread(path)`` (``IMREAD_COLOR``) returns out, byte for
byte, as uint8 [H, W, 3] BGR CUDA tensors.

The host parses each stream's markers (SOI, APPn -- the Exif orientation of APP1 and the Adobe transform of APP14 --,
DQT, DHT, SOF0 / SOF1, DRI, SOS, RSTn, EOI), builds libjpeg's derived Huffman tables and one job table per batch, and
uploads them with the compressed bytes in one pinned staging copy.  The device decodes 8-bit sequential Huffman
streams with one interleaved scan of 1 or 3 components, sampled 4:4:4, 4:2:2, 4:2:0, 4:4:0 or 4:1:1, with any restart
interval (``ryolo_jpeg_decode``; the arithmetic is in ``csrc/jpeg.cuh``).  Every other stream -- progressive,
arithmetic-coded, 12-bit, lossless, CMYK / YCCK, multi-scan, or one the parser does not accept -- is decoded on the
host by ``cv2.imdecode`` and uploaded into the same output slot, and so is a stream the device finds corrupt or
whose coefficients leave the range where libjpeg-turbo's C and SIMD IDCTs agree.  The route each image took is
returned with it."""
import functools

import numpy as np
import torch

from . import _lib
from .preprocess import _pinned, _staging

DEFAULT_CHUNK_BYTES = 128
DEVICE = "device"
YCC, RGB, GRAY = 0, 1, 2                  # RYOLO_JPEG_YCC / RGB / GRAY
ST_BAD_CODE, ST_TRUNCATED, ST_NO_SYNC, ST_RANGE = 1, 2, 4, 8      # RYOLO_JPEG_ST_*

_NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                     13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                     45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)
# sampling ratios (hmax / h, vmax / v) the device upsamples: full size, h2v1, h1v2, h2v2 (fancy), h4v1 (box)
_RATIOS = {(1, 1), (2, 1), (1, 2), (2, 2), (4, 1)}
_SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "hierarchical", 0xC6: "hierarchical progressive",
              0xC7: "hierarchical lossless", 0xC9: "arithmetic", 0xCA: "arithmetic progressive",
              0xCB: "arithmetic lossless", 0xCD: "arithmetic hierarchical", 0xCE: "arithmetic hierarchical",
              0xCF: "arithmetic hierarchical"}

IMAGE_DTYPE = np.dtype(_lib.JpegImage)
SEGMENT_DTYPE = np.dtype(_lib.JpegSegment)
HUFF_DTYPE = np.dtype(_lib.JpegHuff)


class Unsupported(Exception):
    """the stream goes to the host decoder; the message says why"""


class Header:
    """What the parser takes from one stream: frame, tables, scan and the entropy-coded segments."""
    __slots__ = ("width", "height", "ncomp", "color", "h", "v", "hmax", "vmax", "mcux", "mcuy", "bpm", "quant",
                 "dc", "ac", "restart", "segments", "orient", "out_hw")


def _u16(d, i):
    return (int(d[i]) << 8) | int(d[i + 1])


@functools.lru_cache(maxsize=256)
def derived_table(counts, vals, is_dc):
    """libjpeg's jpeg_make_d_derived_tbl for one DHT table (counts: 16 code counts, vals: the symbols, both bytes) as a
    ryolo_jpeg_huff record: the 9-bit lookahead, maxcode and valoff per length, and the symbols.  Raises Unsupported
    where libjpeg rejects the table."""
    counts = np.frombuffer(counts, np.uint8).astype(np.int64)
    vals = np.frombuffer(vals, np.uint8)
    if counts.sum() > 256 or counts.sum() != len(vals):
        raise Unsupported("bad Huffman table")
    if is_dc and len(vals) and vals.max() > 15:
        raise Unsupported("bad Huffman table")
    rec = np.zeros((), HUFF_DTYPE)
    code, p = 0, 0
    lut = rec["lut"]
    for length in range(1, 17):
        n = int(counts[length - 1])
        if n:
            rec["valoff"][length] = p - code
            for i in range(n):
                if length <= 9:
                    lo = (code + i) << (9 - length)
                    lut[lo:lo + (1 << (9 - length))] = (length << 8) | int(vals[p + i])
            code += n
            p += n
            rec["maxcode"][length] = code - 1
        else:
            rec["maxcode"][length] = -1
        if code > (1 << length):
            raise Unsupported("bad Huffman table")
        code <<= 1
    rec["maxcode"][17] = 0xFFFFF
    rec["vals"][:len(vals)] = vals
    return rec


def _exif_orientation(seg):
    """the orientation tag (0x0112) of IFD0 of an APP1 Exif payload as cv2 reads it: 1..8, 1 when absent or out of
    range.  Raises Unsupported for anything it cannot read exactly."""
    if bytes(seg[:6]) != b"Exif\0\0":
        raise Unsupported("APP1 that is not Exif")
    t = bytes(seg[6:])
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        raise Unsupported("malformed Exif")
    bo = "little" if t[:2] == b"II" else "big"
    rd = lambda o, n: int.from_bytes(t[o:o + n], bo)
    if rd(2, 2) != 42:
        raise Unsupported("malformed Exif")
    ifd = rd(4, 4)
    if ifd + 2 > len(t) or ifd + 2 + 12 * rd(ifd, 2) > len(t):
        raise Unsupported("malformed Exif")
    for e in range(rd(ifd, 2)):
        o = ifd + 2 + 12 * e
        if rd(o, 2) == 0x0112:
            if rd(o + 2, 2) != 3 or rd(o + 4, 4) != 1:
                raise Unsupported("unusual Exif orientation entry")
            val = rd(o + 8, 2)
            return val if 1 <= val <= 8 else 1
    return 1


def parse(d):
    """Parse one JPEG stream (uint8 array).  Returns a Header for a stream the device decodes; raises Unsupported (with
    the reason) for one the host decodes."""
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Unsupported("not a JPEG stream")
    hd = Header()
    quant, huff, frame = {}, {}, None
    restart, jfif, adobe, orient, app1_seen = 0, False, None, 1, False
    i = 2
    while True:
        if i < n and d[i] != 0xFF:
            raise Unsupported("bytes between markers")
        while i < n and d[i] == 0xFF:
            i += 1
        if i >= n:
            raise Unsupported("no scan")
        m = int(d[i])
        i += 1
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7:
            raise Unsupported("unexpected marker 0x%02X" % m)
        if m == 0xD9:
            raise Unsupported("no scan")
        if i + 2 > n:
            raise Unsupported("truncated header")
        ln = _u16(d, i)
        if ln < 2 or i + ln > n:
            raise Unsupported("truncated header")
        seg = d[i + 2:i + ln]
        i += ln
        if m == 0xE0 and ln >= 16 and bytes(seg[:5]) == b"JFIF\0":     # libjpeg: APP0_DATA_LEN 14
            jfif = True
        elif m == 0xE1 and not app1_seen:                  # cv2 reads the first APP1 as Exif
            app1_seen = True
            orient = _exif_orientation(seg)
        elif m == 0xEE and ln >= 14 and bytes(seg[:5]) == b"Adobe":     # APP14_DATA_LEN 12
            adobe = int(seg[11])
        elif m == 0xDB:
            k = 0
            while k < len(seg):
                pq, tq = int(seg[k]) >> 4, int(seg[k]) & 15
                sz = 128 if pq else 64
                if tq > 3 or pq > 1 or k + 1 + sz > len(seg):
                    raise Unsupported("bad DQT")
                raw = seg[k + 1:k + 1 + sz]
                vals = raw.view(">u2").astype(np.int64) if pq else raw.astype(np.int64)
                if vals.max() > 32767:
                    raise Unsupported("16-bit quantisation value above 32767")
                q = np.zeros(64, np.uint16)
                q[_NATURAL] = vals
                quant[tq] = q
                k += 1 + sz
        elif m == 0xC4:
            k = 0
            while k < len(seg):
                tc, th = int(seg[k]) >> 4, int(seg[k]) & 15
                if k + 17 > len(seg) or tc > 1 or th > 3:
                    raise Unsupported("bad DHT")
                counts = seg[k + 1:k + 17]
                cnt = int(counts.astype(np.int64).sum())
                if cnt > 256 or k + 17 + cnt > len(seg):
                    raise Unsupported("bad DHT")
                huff[(tc, th)] = (bytes(counts), bytes(seg[k + 17:k + 17 + cnt]))
                k += 17 + cnt
        elif m == 0xDD:
            if len(seg) != 2:
                raise Unsupported("bad DRI")
            restart = _u16(seg, 0)
        elif m in (0xC0, 0xC1):
            if frame is not None or len(seg) < 6:
                raise Unsupported("bad SOF")
            prec, hgt, wid, nf = int(seg[0]), _u16(seg, 1), _u16(seg, 3), int(seg[5])
            if prec != 8:
                raise Unsupported("%d-bit samples" % prec)
            if nf not in (1, 3) or len(seg) != 6 + 3 * nf:
                raise Unsupported("%d components" % nf)
            if hgt == 0 or wid == 0:
                raise Unsupported("frame height or width 0")
            frame = [(int(seg[6 + 3 * c]), int(seg[7 + 3 * c]) >> 4, int(seg[7 + 3 * c]) & 15, int(seg[8 + 3 * c]))
                     for c in range(nf)]
            hd.width, hd.height, hd.ncomp = wid, hgt, nf
        elif m in _SOF_NAMES:
            raise Unsupported(_SOF_NAMES[m])
        elif m in (0xDC, 0xCC, 0xDE, 0xDF):
            raise Unsupported("marker 0x%02X" % m)
        elif m == 0xDA:
            if frame is None:
                raise Unsupported("SOS before SOF")
            ns = int(seg[0]) if len(seg) else 0
            if len(seg) != 4 + 2 * ns or ns != len(frame):
                raise Unsupported("not one interleaved scan of every component")
            ids = [int(seg[1 + 2 * c]) for c in range(ns)]
            if ids != [f[0] for f in frame]:
                raise Unsupported("scan components not in frame order")
            ss, se, ahl = int(seg[1 + 2 * ns]), int(seg[2 + 2 * ns]), int(seg[3 + 2 * ns])
            if ss != 0 or se != 63 or ahl != 0:
                raise Unsupported("spectral selection in a sequential scan")
            tabs = [(int(seg[2 + 2 * c]) >> 4, int(seg[2 + 2 * c]) & 15) for c in range(ns)]
            _frame(hd, frame, quant, huff, tabs, restart, jfif, adobe)
            hd.segments = _segments(d, i, hd)
            hd.orient = orient
            hd.out_hw = (hd.width, hd.height) if orient >= 5 else (hd.height, hd.width)
            return hd
        # other APPn, COM: skipped


def _frame(hd, frame, quant, huff, tabs, restart, jfif, adobe):
    nf = hd.ncomp
    hs, vs = [f[1] for f in frame], [f[2] for f in frame]
    if min(hs + vs) < 1 or max(hs + vs) > 4:
        raise Unsupported("bad sampling factors")
    if nf == 1:
        hs, vs = [1], [1]                                  # one component: the MCU is one block
    hd.hmax, hd.vmax = max(hs), max(vs)
    for h, v in zip(hs, vs):
        if hd.hmax % h or hd.vmax % v or (hd.hmax // h, hd.vmax // v) not in _RATIOS:
            raise Unsupported("sampling %s" % ",".join("%dx%d" % hv for hv in zip(hs, vs)))
    hd.h, hd.v = hs, vs
    hd.bpm = sum(h * v for h, v in zip(hs, vs))
    if hd.bpm > 10:
        raise Unsupported("more than 10 blocks per MCU")
    hd.mcux = -(-hd.width // (8 * hd.hmax))
    hd.mcuy = -(-hd.height // (8 * hd.vmax))
    if nf == 1:
        hd.color = GRAY
    else:
        ids = [f[0] for f in frame]
        rgb = (not jfif and adobe == 0) or (not jfif and adobe is None and ids == [82, 71, 66])
        hd.color = RGB if rgb else YCC
    hd.quant, hd.dc, hd.ac = [], [], []
    for (cid, _, _, tq), (td, ta) in zip(frame, tabs):
        if tq not in quant:
            raise Unsupported("quantisation table %d not defined" % tq)
        if (0, td) not in huff or (1, ta) not in huff:
            raise Unsupported("Huffman table not defined")
        hd.quant.append(quant[tq])
        hd.dc.append(derived_table(*huff[(0, td)], True))
        hd.ac.append(derived_table(*huff[(1, ta)], False))
    hd.restart = restart


def _segments(d, start, hd):
    """the entropy-coded segments of the scan that starts at byte `start`: [(start, end, first_mcu, nmcu)], split at
    the restart markers, which must come in sequence; the scan must end at EOI or at the end of the stream"""
    n = len(d)
    ff = np.flatnonzero(d[start:n - 1] == 0xFF) + start
    nxt = d[ff + 1]
    marks = ff[nxt != 0]
    codes = d[marks + 1].astype(np.int64)
    is_rst = (codes >= 0xD0) & (codes <= 0xD7)
    stop = np.flatnonzero(~is_rst)
    if not len(stop):
        raise Unsupported("no EOI")
    end = int(marks[stop[0]])
    rst = marks[:stop[0]]
    if int(d[end + 1]) != 0xD9:
        raise Unsupported("more than one scan" if int(d[end + 1]) != 0xFF else "fill bytes in the scan")
    total = hd.mcux * hd.mcuy
    ri = hd.restart if hd.restart else total
    nseg = -(-total // ri)
    if len(rst) != nseg - 1 or np.any(d[rst + 1] != 0xD0 + np.arange(len(rst)) % 8):
        raise Unsupported("restart markers out of sequence")
    starts = np.concatenate([[start], rst + 2]).astype(np.int64)
    ends = np.concatenate([rst, [end]]).astype(np.int64)
    first = np.arange(nseg, dtype=np.int64) * ri
    return starts, ends, first, np.minimum(ri, total - first)


def _fallback(d, i):
    import cv2
    img = cv2.imdecode(d, cv2.IMREAD_COLOR)
    if img is None:
        raise ValueError("decode_images: image %d is not an image cv2 can decode" % i)
    return img


class Layout:
    """The host half of a batch, without a device: the parsed streams, the route of each, the host decodes, the output
    offsets and, when any stream goes to the device, the staging bytes (job tables, Huffman and quantisation tables,
    compressed bytes) with the launch arguments."""

    def __init__(self, blobs, chunk_bytes=DEFAULT_CHUNK_BYTES):
        self.chunk_bytes = int(chunk_bytes)
        if self.chunk_bytes < 1:
            raise ValueError("decode_images: chunk_bytes must be >= 1")
        self.arrays, self.heads, self.routes, self.host = [], [], [], {}
        for i, b in enumerate(blobs):
            a = np.frombuffer(b, np.uint8) if isinstance(b, (bytes, bytearray, memoryview)) else np.asarray(b)
            if a.dtype != np.uint8 or a.ndim != 1:
                raise ValueError("decode_images: blob %d must be bytes or a 1-D uint8 array" % i)
            self.arrays.append(a)
            try:
                self.heads.append(parse(a))
                self.routes.append(DEVICE)
            except Unsupported as e:
                self.heads.append(None)
                self.routes.append("host: %s" % e)
                self.host[i] = _fallback(a, i)
        self.shapes = [(h.out_hw if h is not None else self.host[i].shape[:2]) for i, h in enumerate(self.heads)]
        self.out_offs = np.zeros(len(self.shapes) + 1, np.int64)
        self.out_offs[1:] = np.cumsum([_align(3 * hh * ww) for hh, ww in self.shapes])
        self.dev_idx = [i for i, h in enumerate(self.heads) if h is not None]
        self.stage = None
        if self.dev_idx:
            self._tables()

    def _tables(self):
        heads = [self.heads[i] for i in self.dev_idx]
        imgs = np.zeros(len(heads), IMAGE_DTYPE)
        huffs, hkey, quants, qkey = [], {}, [], {}
        seg_parts, data_off, area = [], 0, 0
        for j, (i, hd) in enumerate(zip(self.dev_idx, heads)):
            r = imgs[j]
            r["out_off"] = self.out_offs[i]
            r["width"], r["height"], r["out_h"], r["out_w"] = hd.width, hd.height, hd.out_hw[0], hd.out_hw[1]
            r["orient"], r["ncomp"], r["color"] = hd.orient, hd.ncomp, hd.color
            r["hmax"], r["vmax"], r["mcux"], r["mcuy"], r["bpm"] = hd.hmax, hd.vmax, hd.mcux, hd.mcuy, hd.bpm
            r["coef_off"] = area
            area += _align(128 * hd.mcux * hd.mcuy * hd.bpm, 256)
            r["boff"][:] = 64
            r["h"][:] = r["v"][:] = 1
            boff = 0
            for c in range(hd.ncomp):
                h, v = hd.h[c], hd.v[c]
                r["h"][c], r["v"][c], r["boff"][c] = h, v, boff
                boff += h * v
                r["pitch"][c] = hd.mcux * h * 8
                r["dw"][c] = -(-hd.width * h // hd.hmax)
                r["dh"][c] = -(-hd.height * v // hd.vmax)
                r["plane_off"][c] = area
                area += _align(int(r["pitch"][c]) * hd.mcuy * v * 8, 256)
                for tab, field in ((hd.dc[c], "dctab"), (hd.ac[c], "actab")):
                    k = tab.tobytes()
                    if k not in hkey:
                        hkey[k] = len(huffs)
                        huffs.append(tab)
                    r[field][c] = hkey[k]
                k = hd.quant[c].tobytes()
                if k not in qkey:
                    qkey[k] = 64 * len(quants)
                    quants.append(hd.quant[c])
                r["qtab"][c] = qkey[k]
            starts, ends, first, nmcu = hd.segments
            seg_parts.append((starts + data_off, ends + data_off, first, nmcu, j))
            data_off += _align(len(self.arrays[i]))
        segs = np.zeros(sum(len(p[0]) for p in seg_parts), SEGMENT_DTYPE)
        k = 0
        for starts, ends, first, nmcu, j in seg_parts:
            s = segs[k:k + len(starts)]
            s["start"], s["end"], s["first_mcu"], s["nmcu"], s["image"] = starts, ends, first, nmcu, j
            k += len(starts)
        nchunk = np.maximum(1, -(-(segs["end"] - segs["start"]) // self.chunk_bytes))
        segs["nchunk"] = nchunk
        segs["first_chunk"] = np.concatenate([[0], np.cumsum(nchunk)[:-1]])
        chunk_seg = np.repeat(np.arange(len(segs), dtype=np.int32), nchunk)
        if len(chunk_seg) >= 2 ** 31 - 1 or data_off >= 2 ** 32 - 8:
            raise ValueError("decode_images: batch too large (%d chunks, %d bytes)" % (len(chunk_seg), data_off))
        parts = [imgs.view(np.uint8), segs.view(np.uint8), chunk_seg.view(np.uint8),
                 np.array(huffs, HUFF_DTYPE).view(np.uint8), np.concatenate(quants).view(np.uint8)]
        at, self.offsets = 0, []
        for p in parts:
            self.offsets.append(at)
            at = _align(at + p.nbytes, 256)
        self.offsets.append(at)                            # the compressed bytes
        self.stage = np.zeros(at + data_off, np.uint8)
        for o, p in zip(self.offsets, parts):
            self.stage[o:o + p.nbytes] = p
        pos = at
        for i in self.dev_idx:
            a = self.arrays[i]
            self.stage[pos:pos + len(a)] = a
            pos += _align(len(a))
        self.nimg, self.nsegs, self.nchunks, self.data_bytes = len(heads), len(segs), len(chunk_seg), data_off
        self.max_blocks = max(hd.mcux * hd.mcuy * hd.bpm for hd in heads)
        self.max_out_h = max(hd.out_hw[0] for hd in heads)
        self.area = area


class Batch:
    """One batch staged on the device: decode() issues the kernels on the current stream and may be replayed or
    captured in a CUDA graph while the batch is kept."""

    def __init__(self, blobs, device, chunk_bytes=DEFAULT_CHUNK_BYTES, out=None):
        self.device = device
        self.lay = lay = Layout(blobs, chunk_bytes)
        self.routes = list(lay.routes)
        total_out = int(lay.out_offs[-1])
        if out is None:
            out = torch.empty(total_out, dtype=torch.uint8, device=device)
        elif (not out.is_cuda or out.device != device or out.dtype != torch.uint8 or not out.is_contiguous()
              or out.numel() < total_out):
            raise ValueError("decode_images: out must be a contiguous uint8 CUDA tensor of >= %d bytes on %s"
                             % (total_out, device))
        self.out = out.view(-1)
        self.images = [self.out[int(o):int(o) + 3 * hh * ww].view(hh, ww, 3)
                       for o, (hh, ww) in zip(lay.out_offs, lay.shapes)]
        self.staged_bytes = 0
        if lay.stage is not None:
            n = lay.stage.nbytes
            pinned = _pinned(device, n)
            pinned[:n].numpy()[:] = lay.stage
            self.tables = torch.empty(n, dtype=torch.uint8, device=device)
            self.tables.copy_(pinned[:n], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            _staging[device.index] = (pinned, ev)
            self.ptrs = [self.tables.data_ptr() + o for o in lay.offsets]
            ws = _lib.lib.ryolo_jpeg_workspace_bytes(lay.nchunks, lay.area)
            self.workspace = torch.empty(ws, dtype=torch.uint8, device=device)
            self.status = torch.zeros(lay.nimg, dtype=torch.int32, device=device)
            self.staged_bytes = n

    def decode(self, stages=3):
        """issue the device decode of the staged images on the current stream (stages: 1 entropy, 2 pixels, 3 both)"""
        lay = self.lay
        if lay.stage is None:
            return
        p = self.ptrs
        st = _lib.lib.ryolo_jpeg_decode(p[0], lay.nimg, p[1], lay.nsegs, p[2], lay.nchunks, lay.chunk_bytes, p[5],
                                        lay.data_bytes, p[3], p[4], lay.max_blocks, lay.max_out_h,
                                        _lib.ptr(self.out), _lib.ptr(self.status), _lib.ptr(self.workspace),
                                        self.workspace.numel(), lay.area, stages, _lib.stream_ptr(self.device))
        _lib.check(st, "ryolo_jpeg_decode")

    def finish(self):
        """upload the host-decoded images, read the device status once and decode the images it rejects on the host"""
        lay = self.lay
        for i, img in lay.host.items():
            self.images[i].copy_(torch.from_numpy(np.ascontiguousarray(img)))
        if lay.stage is not None:
            status = self.status.cpu().numpy()
            for j in np.flatnonzero(status):
                i = lay.dev_idx[int(j)]
                img = _fallback(lay.arrays[i], i)
                if tuple(img.shape) != tuple(self.images[i].shape):
                    raise ValueError("decode_images: image %d decodes to %s on the host, its header says %s"
                                     % (i, img.shape, tuple(self.images[i].shape)))
                self.images[i].copy_(torch.from_numpy(img))
                self.routes[i] = "host: %s (status %d)" % (status_reason(int(status[j])), int(status[j]))
        return self.images, self.routes


def status_reason(st):
    """why the device handed an image back, from its RYOLO_JPEG_ST_* mask"""
    if st & (ST_BAD_CODE | ST_TRUNCATED | ST_NO_SYNC):
        return "corrupt entropy-coded data"
    return "coefficients outside the IDCT's exact range"


def _align(n, a=16):
    return (n + a - 1) // a * a


def decode_images(blobs, device=None, out=None, chunk_bytes=DEFAULT_CHUNK_BYTES):
    """Decode a batch of JPEG files on the device, byte for byte as ``cv2.imread(path)`` decodes them.

    blobs: list of file contents, ``bytes`` or 1-D uint8 numpy arrays (``np.fromfile(path, np.uint8)``).
    out: optional uint8 CUDA tensor the images are written into (large enough for all of them, each aligned to 16
    bytes).  chunk_bytes: the entropy decoder's chunk size (one GPU thread per chunk; smaller chunks, more threads).
    Returns (images, routes): images a list of uint8 [H, W, 3] BGR CUDA tensors, views into one buffer, in the Exif
    orientation; routes a list of "device" or "host: <reason>" per image.  A stream cv2 cannot decode raises
    ValueError."""
    if not isinstance(blobs, (list, tuple)) or len(blobs) == 0 or len(blobs) > 65535:
        raise ValueError("decode_images: blobs must be a list of 1 to 65535 JPEG file contents")
    if device is None:
        device = out.device if out is not None else torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("decode_images runs on a CUDA device only, got %s" % (device,))
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        batch = Batch(blobs, device, chunk_bytes, out)
        batch.decode()
        return batch.finish()
