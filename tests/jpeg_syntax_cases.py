"""Seeded JPEG streams that cv2 never writes, made with tests/jpeg_writer.py, for the decoder tests: dequantised
coefficients far outside what 8-bit pixels produce, DC sums that leave int16, unusual Huffman tables and EOB / ZRL
sequences, byte stuffing on chunk boundaries, every colour rule, and samplings cv2 cannot write.

Each case is (name, blob, expect): "device" (decoded on the device), "range" (the device hands it to the host with
RYOLO_JPEG_ST_RANGE), "host" (the parser or the entropy decoder sends it to the host) or "any" (either way).  Whatever
the route, the image must equal cv2's; a stream cv2 rejects must be rejected."""
import numpy as np

import jpeg_writer as jw
from jpeg_cases import encode, picture

YCC3 = [{"id": 1, "h": 1, "v": 1, "tq": 0, "td": 0, "ta": 0}, {"id": 2, "h": 1, "v": 1, "tq": 0, "td": 0, "ta": 0},
        {"id": 3, "h": 1, "v": 1, "tq": 0, "td": 0, "ta": 0}]


def _full(symbols):
    f = np.zeros(256, np.int64)
    f[list(symbols)] = 1
    return jw.huff_from_freqs(f)


# tables with a code for every baseline symbol: DC categories 0..11, AC (run, size) for sizes 1..10, EOB and ZRL
FULL_DC = _full(range(12))
FULL_AC = _full([0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)])


def natural_stream(seed=0, h=40, w=56, sampling="444", quality=100):
    """(width, height, comps, blocks, quant, dc, ac, restart) of a cv2-written stream"""
    return jw.read_cv2_stream(encode(picture(seed, h, w), quality, sampling))


def surgery(blob, value):
    """blob with every 8-bit quantisation value set to `value` (1..255); the entropy-coded data as cv2 wrote it"""
    b = bytearray(blob)
    i = 2
    while b[i + 1] != 0xDA:
        ln = (b[i + 2] << 8) | b[i + 3]
        if b[i + 1] == 0xDB:
            k = i + 4
            while k < i + 2 + ln:
                assert b[k] >> 4 == 0
                b[k + 1:k + 65] = bytes([value]) * 64
                k += 65
        i += 2 + ln
    return bytes(b)


def _write_opt(width, height, comps, blocks, quant, restart=0, **kw):
    comps, dc, ac = jw.optimal_tables(width, height, comps, blocks, restart)
    return jw.write(width, height, comps, blocks, quant, dc, ac, restart=restart, **kw)


def qtable_cases():
    """the reproducer: a q100 4:4:4 40 x 56 stream with its quantisation tables rewritten, entropy data untouched"""
    base = encode(picture(0, 40, 56), 100, "444")
    out = []
    for v in (2, 4):
        out.append(("qsurgery_8bit_%d" % v, surgery(base, v), "any"))
    for v in (8, 16, 32, 64, 128, 255):
        out.append(("qsurgery_8bit_%d" % v, surgery(base, v), "range"))
    w, h, comps, blocks, _, dc, ac, _ = jw.read_cv2_stream(base)
    for v in (1000, 32767):
        q = {s: [v] * 64 for s in {c["tq"] for c in comps}}
        out.append(("qsurgery_16bit_%d" % v, jw.write(w, h, comps, blocks, q, dc, ac, sixteen=True, sof1=True),
                    "range"))
    return out


def magnitude_cases():
    """per-block largest dequantised |coef * q| from 2^9 to 2^20 on a 64 x 64 4:4:4 frame of 64 blocks per component:
    block k holds its value at zigzag k alone (k = 0: the DC alone); plus a frame of dense random blocks.  8-bit
    tables up to q 255, then 16-bit tables with SOF1."""
    r = np.random.default_rng(17)
    out = []
    for e in range(9, 21):
        mag = 1 << e
        q = max(1, mag >> 10)
        coef = mag // q
        quant = {0: [q] * 64}
        wide = q > 255
        blocks = [np.zeros((8, 8, 64), np.int64) for _ in range(3)]
        for ci in range(3):
            for k in range(64):
                blocks[ci][k // 8, k % 8, k] = coef if (k + ci) % 2 == 0 else -coef
        out.append(("mag_single_2^%d" % e, _write_opt(64, 64, [dict(c) for c in YCC3], blocks, quant, sixteen=wide,
                                                      sof1=wide), "any"))
        dense = [r.integers(-coef, coef + 1, (8, 8, 64)) // np.arange(1, 65) ** 0.5 for _ in range(3)]
        dense = [d.astype(np.int64) for d in dense]
        out.append(("mag_dense_2^%d" % e, _write_opt(64, 64, [dict(c) for c in YCC3], dense, quant, sixteen=wide,
                                                     sof1=wide), "any"))
    return out


def dc_sum_cases():
    """runs of +-2047 DC differences on a one-component 8 x 512 frame (64 blocks) that carry the running sum past
    int16, with and without restart intervals that reset it; q 1"""
    out = []
    one = [{"id": 1, "h": 1, "v": 1, "tq": 0, "td": 0, "ta": 0}]
    for sign in (1, -1):
        for rst in (0, 5, 32):
            b = np.zeros((1, 64, 64), np.int64)
            b[0, :, 0] = sign * 2047 * np.arange(1, 65)
            if rst:                                            # each restart interval starts its sum from zero
                b[0, :, 0] = sign * 2047 * (np.arange(64) % rst + 1)
            expect = "range"
            out.append(("dc_sum_%s_rst%d" % ("up" if sign > 0 else "down", rst),
                        _write_opt(512, 8, [dict(c) for c in one], [b], {0: [1] * 64}, restart=rst), expect))
    return out


def _natural_blocks():
    w, h, comps, blocks, quant, dc, ac, _ = natural_stream(3, 32, 48, "444", 90)
    return w, h, comps, blocks, quant


def huffman_cases():
    out = []
    w, h, comps, blocks, quant = _natural_blocks()
    comps, dc, ac = jw.optimal_tables(w, h, comps, blocks)
    # every code length 1..16: one code of each length 1..15 and one of 16 bits, over blocks with 16 AC symbols
    r = np.random.default_rng(21)
    syms16 = [0x00, 0xF0, 0x02, 0x03] + [(k << 4) | 1 for k in range(12)]
    few = [np.zeros_like(b) for b in blocks]
    for bl in few:
        for blk in bl.reshape(-1, 64):
            blk[0] = r.integers(-40, 40)
            k = 1
            while k < 64:
                k += int(r.choice([0, 1, 2, 5, 11, 17, 27]))
                if k < 64:
                    blk[k] = int(r.choice([-1, 1]))
                k += 1
    assert {s_ for bl in few for blk in bl.reshape(-1, 64) for s_, _, _ in jw.block_symbols(blk)} <= set(syms16)
    c1 = [dict(c, td=0, ta=0) for c in comps]
    lengths = (bytes([1] * 16), bytes(syms16))
    out.append(("huff_lengths_1_to_16", jw.write(w, h, c1, few, quant, {0: FULL_DC}, {0: lengths}), "device"))
    used = sorted(set(s_ for ci in range(3) for s_ in ac[ci][1]))
    dsyms = sorted(set(s_ for ci in range(3) for s_ in dc[ci][1]))
    dtab = (bytes([0] * 15 + [len(dsyms)]), bytes(dsyms))
    all16 = (bytes([0] * 15 + [len(used)]), bytes(used))
    out.append(("huff_all_16bit", jw.write(w, h, c1, blocks, quant, {0: dtab}, {0: all16}), "device"))
    # tables in slots 2 and 3, one per component, and a table with one symbol (a flat gray frame: DC 0, EOB)
    c23 = [dict(c, td=2 + (i > 0), ta=3 - (i > 0)) for i, c in enumerate(comps)]
    fa = np.zeros(256, np.int64)
    fa[used] = 1
    out.append(("huff_slots_2_3", jw.write(w, h, c23, blocks, quant, {2: dc[0], 3: dtab}, {3: ac[0], 2: jw.huff_from_freqs(fa)}),
                "any"))
    flat = [np.zeros_like(b) for b in blocks]
    one_sym = (bytes([1] + [0] * 15), bytes([0]))
    out.append(("huff_one_symbol", jw.write(w, h, [dict(c, td=0, ta=0) for c in comps], flat, quant, {0: one_sym},
                                            {0: one_sym}), "device"))
    # category-11 DC and category-10 AC codes at q 1 (values kept inside the IDCT's range by their neighbours)
    big = [np.zeros_like(b) for b in blocks]
    big[0][0, 0, 0] = 2047 // 2
    big[0][0, 1, 0] = -1023
    big[1][1, 1, 5] = 700
    big[2][2, 2, 9] = -1023 // 2
    big[2][2, 3, 0], big[2][2, 4, 0] = 1023, -1024       # DC differences of category 11
    out.append(("huff_cat11_dc_cat10_ac", _write_opt(w, h, [dict(c) for c in comps], big, {0: [1] * 64, 1: [1] * 64}),
                "any"))
    return out


def eob_zrl_cases():
    """blocks that end at zigzag 63 without EOB, a run reaching 63, ZRL landing on 48 then EOB, and a ZRL that passes
    64 (libjpeg accepts it and stops the block; the device sends the stream to the host)"""
    w, h, comps, blocks, quant = _natural_blocks()
    blocks = [b.copy() for b in blocks]
    blocks[0][0, 0, 63] = 3                                # nonzero 63: no EOB
    blocks[0][0, 1, 1:] = 0
    blocks[0][0, 1, 63] = -2                               # a run of 61 zeros reaching 63
    zrl48 = [(0x01, 1), (0xF0, 0), (0xF0, 0), (0xF0, 0), (0x00, 0)]      # 1, then zeros to 48, then EOB
    comps2, dc, ac = [dict(c, td=0, ta=0) for c in comps], {0: FULL_DC}, {0: FULL_AC}
    out = [("zrl_ends_at_63_and_run_to_63", jw.write(w, h, comps2, blocks, quant, dc, ac), "device"),
           ("zrl_to_48_then_eob", jw.write(w, h, comps2, blocks, quant, dc, ac, ac_symbols={(0, 2, 2): zrl48}),
            "device")]
    past = [(0x01, 1), (0xF0, 0), (0xF0, 0), (0xF0, 0), (0xF0, 0)]       # 1 + 64 zeros: past the block
    out.append(("zrl_past_64", jw.write(w, h, comps2, blocks, quant, dc, ac, ac_symbols={(0, 2, 2): past}), "host"))
    return out


def stuffing_cases():
    """streams dense in 0xFF bytes (DC differences of -1 with a table whose codes are all ones), so 0xFF00 stuffing
    falls on every chunk boundary for small chunks"""
    w, h = 48, 32
    b = [np.zeros((4, 6, 64), np.int64) for _ in range(3)]
    r = np.random.default_rng(5)
    for ci in range(3):
        b[ci][..., 0] = -np.arange(24).reshape(4, 6)       # difference -1 per block: extra bit 0, then the code
        b[ci][..., 1] = r.integers(-1, 2, (4, 6))
    ac = (bytes([0, 0, 0, 0, 0, 0, 0, 3] + [0] * 8), bytes([0x00, 0x01, 0x02]))
    dc = (bytes([0] * 7 + [2] + [0] * 8), bytes([1, 0]))   # category 1 -> 0xFE... code 0, category 0 -> code 1
    comps = [dict(c) for c in YCC3]
    out = [("stuffing_dense_ff", jw.write(w, h, comps, b, {0: [2] * 64}, {0: dc}, {0: ac}), "device")]
    return out


def colour_cases():
    """every combination of JFIF / Adobe 0 / 1 / 2 / no APP segment with component ids 1-2-3, 'R','G','B' and others:
    the colour space libjpeg-turbo's default_decompress_parms picks, as cv2 decodes it"""
    w, h, comps, blocks, quant, dc, ac, _ = natural_stream(5, 24, 40, "444", 90)
    out = []
    for app_name, app in (("none", ()), ("jfif", ("jfif",)), ("adobe0", (("adobe", 0),)), ("adobe1", (("adobe", 1),)),
                          ("adobe2", (("adobe", 2),)), ("jfif_adobe0", ("jfif", ("adobe", 0)))):
        for ids_name, ids in (("123", (1, 2, 3)), ("RGB", (82, 71, 66)), ("other", (5, 9, 200)), ("012", (0, 1, 2))):
            c = [dict(x, id=i) for x, i in zip(comps, ids)]
            expect = "device"                              # Adobe 2 (YCCK) with 3 components: libjpeg warns, YCbCr
            out.append(("colour_%s_%s" % (app_name, ids_name), jw.write(w, h, c, blocks, quant, dc, ac, app=app),
                        expect))
    return out


def expected_color(name):
    """the colour space libjpeg-turbo 3.1 picks (jdapimin.c default_decompress_parms) for colour_<app>_<ids>, as
    decode.YCC / RGB: JFIF means YCbCr; else an Adobe transform 0 means RGB and any other YCbCr; else component ids
    'R','G','B' mean RGB; else YCbCr"""
    app, ids = name[len("colour_"):].rsplit("_", 1)
    if app.startswith("jfif"):
        return 0
    if app.startswith("adobe"):
        return 1 if app == "adobe0" else 0
    return 1 if ids == "RGB" else 0


def sampling_cases():
    """samplings _frame accepts that cv2 cannot write: chroma sampled finer than luma, mixed h2v1 and h4v1, widths of 1
    to 3 samples where fancy upsampling turns into box replication, each at sizes that leave partial MCUs"""
    r = np.random.default_rng(9)
    out = []
    specs = {"chroma_finer_h": [(1, 1), (2, 1), (2, 1)], "chroma_finer_hv": [(1, 1), (2, 2), (2, 2)],
             "mixed_h2_h4": [(4, 1), (2, 1), (1, 1)], "luma_h2v2_cr_h2v1": [(2, 2), (2, 1), (1, 1)],
             "h1v2_only_luma": [(1, 2), (1, 1), (1, 2)], "h4v1_all": [(4, 1), (4, 1), (1, 1)]}
    for name, hv in specs.items():
        for (wd, ht) in ((1, 1), (2, 3), (3, 2), (13, 9), (37, 21)):
            comps = [{"id": i + 1, "h": a, "v": b, "tq": min(i, 1), "td": 0, "ta": 0} for i, (a, b) in enumerate(hv)]
            blocks = []
            for ci in range(3):
                rows, cols = jw.block_grid(wd, ht, comps, ci)
                bl = np.zeros((rows, cols, 64), np.int64)
                bl[..., 0] = r.integers(-60, 60, (rows, cols))
                bl[..., 1:6] = r.integers(-8, 9, (rows, cols, 5))
                blocks.append(bl)
            quant = {0: [4] * 64, 1: [6] * 64}
            out.append(("sampling_%s_%dx%d" % (name, wd, ht), _write_opt(wd, ht, comps, blocks, quant), "any"))
    return out


def marker_order_cases():
    """tables after SOF, and a quantisation / Huffman table defined twice before SOS: the last definition wins"""
    w, h, comps, blocks, quant, dc, ac, _ = natural_stream(6, 24, 32, "420", 85)
    decoys = [jw.dqt(s, [99] * 64) for s in quant] + [jw.dht(1, s, (bytes([0, 2] + [0] * 14), bytes([0, 1])))
                                                      for s in ac]
    return [("order_sof_first", jw.write(w, h, comps, blocks, quant, dc, ac, order=("sof", "dht", "dqt", "dri")),
             "device"),
            ("order_tables_redefined", jw.write(w, h, comps, blocks, quant, dc, ac, decoys=decoys), "device"),
            ("order_exif6_dri2", jw.write(w, h, comps, blocks, quant, dc, ac, restart=2, exif=6), "device")]


def all_cases():
    out = []
    for f in (qtable_cases, magnitude_cases, dc_sum_cases, huffman_cases, eob_zrl_cases, stuffing_cases, colour_cases,
              sampling_cases, marker_order_cases):
        out += f()
    return out
