"""Test-side helpers: oracle / reference-build loaders and the seeded input generators of SURVEY.md 8(d).
Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may touch oracle/ -- never the product."""
import ctypes
import math
import os

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
FP = ctypes.POINTER(ctypes.c_float)
I64P = ctypes.POINTER(ctypes.c_int64)
U64P = ctypes.POINTER(ctypes.c_ulonglong)


def P(a):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(FP)


_cache = {}


def oracle():
    if "orc" not in _cache:
        lib = ctypes.CDLL(os.path.join(REPO, "oracle", "librbox_oracle.so"))
        lib.orc_ref_iou.restype = ctypes.c_float
        lib.orc_ref_iou_fma.restype = ctypes.c_float
        lib.orc_skew_iou.restype = ctypes.c_double
        _cache["orc"] = lib
    return _cache["orc"]


def ref_lib(kind):
    """kind in {'host', 'host_fma', 'cuda'}; returns None when oracle/_ref was never built."""
    key = "ref_" + kind
    if key not in _cache:
        path = os.path.join(REPO, "oracle", "_ref", "libref_rnms_%s.so" % kind)
        if os.path.exists(path):
            lib = ctypes.CDLL(path)
            if kind.startswith("host"):
                lib.ref_host_iou.restype = ctypes.c_float
            _cache[key] = lib
        else:
            _cache[key] = None
    return _cache[key]


def gen_boxes(n, seed, canvas=608.0):
    """config-2 generator (SURVEY.md 8d): cx,cy~U[0,canvas), area~U[792,15803), ratio~U[4,9), theta~U(-pi/2,pi/2)."""
    g = torch.Generator().manual_seed(seed)
    cx = torch.rand(n, generator=g) * canvas
    cy = torch.rand(n, generator=g) * canvas
    area = 792 + torch.rand(n, generator=g) * (15803 - 792)
    ratio = 4 + torch.rand(n, generator=g) * 5
    w = (area * ratio).sqrt()
    h = (area / ratio).sqrt()
    th = (torch.rand(n, generator=g) - 0.5) * math.pi
    return torch.stack([cx, cy, w, h, th], 1).float()


def tie_free_scores(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.linspace(0.01, 1, n)[torch.randperm(n, generator=g)].float()


def gen_dets(n, seed, canvas=608.0):
    return torch.cat([gen_boxes(n, seed, canvas), tie_free_scores(n, seed + 1000)[:, None]], 1).contiguous()


def orc_rnms(dets_np, thr, variant=0):
    d = np.ascontiguousarray(dets_np, dtype=np.float32)
    keep = np.empty(len(d), np.int64)
    k = oracle().orc_rnms(P(d), len(d), ctypes.c_float(thr), keep.ctypes.data_as(I64P), variant)
    return keep[:k].copy()


def orc_skew_pairwise(a_np, b_np, mode=0):
    a = np.ascontiguousarray(a_np, dtype=np.float32)
    b = np.ascontiguousarray(b_np, dtype=np.float32)
    out = np.empty((len(a), len(b)), np.float32)
    oracle().orc_skew_iou_pairwise(P(a), len(a), a.shape[1], P(b), len(b), b.shape[1], mode, P(out))
    return out


def orc_skew_paired(a_np, b_np, mode=0):
    a = np.ascontiguousarray(a_np, dtype=np.float32)
    b = np.ascontiguousarray(b_np, dtype=np.float32)
    out = np.empty(len(a), np.float32)
    oracle().orc_skew_iou_paired(P(a), P(b), len(a), a.shape[1], b.shape[1], mode, P(out))
    return out


def adversarial_dets(seed=7):
    """Degenerate NMS inputs: exact duplicates, collinear same-angle neighbours, shared edges, concentric boxes,
    zero-area boxes, NaN box; tie-free scores."""
    base = gen_boxes(96, seed, 120.0)
    rows = [base]
    rows.append(base[:32].clone())                                   # exact duplicates
    sh = base[32:64].clone(); sh[:, 0] += sh[:, 2] * torch.cos(sh[:, 4]); sh[:, 1] += sh[:, 2] * torch.sin(sh[:, 4])
    rows.append(sh)                                                  # shifted by w along own axis: shared short edge
    aa = base[:16].clone(); aa[:, 4] = 0.0; rows.append(aa)           # axis aligned
    ab = aa.clone(); ab[:, 0] += ab[:, 2]; rows.append(ab)            # touching axis-aligned neighbours
    cc = base[64:80].clone(); cc[:, 2:4] *= 0.5; rows.append(cc)      # concentric smaller
    z = base[80:88].clone(); z[:, 2] = 0.0; rows.append(z)            # zero width
    nn_ = base[88:90].clone(); nn_[:, 0] = float("nan"); rows.append(nn_)
    b = torch.cat(rows, 0)
    return torch.cat([b, tie_free_scores(len(b), seed + 1)[:, None]], 1).contiguous()


def filter_edge_rows(nc, conf_thres, min_wh, seed):
    """Decoded rows [n, 6+nc] at the edges of the non_max_suppression candidate filter (utils/nms/nms.py:34-40) and of
    a 4096-bin confidence histogram: conf exactly on bin edges k/4096, one float below and above each; conf == 1.0 in
    many rows; conf == conf_thres and w or h == min_wh (all excluded: strict comparisons) next to the first float above
    each (included); NaN / +inf / -inf in every column in turn, class columns included; tied class maxima (nc > 1)."""
    g = torch.Generator().manual_seed(seed)
    f32 = torch.float32

    def boxes(n):
        b = gen_boxes(n, seed + n, 608.0)
        b[:, 2:4] = min_wh + 1.0 + 60.0 * torch.rand(n, 2, generator=g)
        return b

    def rows(conf):
        """rows whose obj * max(cls) is conf exactly: the maximum class score is 1.0 (twice when nc > 1)"""
        n = len(conf)
        cls = 0.999 * torch.rand(n, nc, generator=g)
        cls[:, 0] = 1.0
        if nc > 1:
            cls[:, nc - 1] = 1.0
        return torch.cat([boxes(n), conf[:, None], cls], 1).to(f32)

    edges = torch.arange(1, 4097, dtype=torch.float64).div(4096).to(f32)
    edges = edges[edges >= conf_thres]
    up = torch.nextafter(edges, torch.full_like(edges, 2.0))
    down = torch.nextafter(edges, torch.zeros_like(edges))
    parts = [rows(edges), rows(up[up <= 1.0]), rows(down), rows(torch.ones(700))]
    thr = torch.tensor([conf_thres], dtype=f32)
    above_thr = torch.nextafter(thr, torch.tensor([2.0]))
    at = rows(thr.repeat(40))
    at[20:, 5] = above_thr                                     # first float above the threshold: included
    parts.append(at)
    wh = rows(torch.full((60,), 0.8))
    wh[:20, 2] = min_wh                                        # w == min_wh: excluded
    wh[20:40, 3] = min_wh                                      # h == min_wh: excluded
    wh[40:50, 2] = torch.nextafter(torch.tensor(float(min_wh)), torch.tensor(1e9))
    wh[50:60, 3] = torch.nextafter(torch.tensor(float(min_wh)), torch.tensor(1e9))
    parts.append(wh)
    for col in range(6 + nc):
        for bad in (float("nan"), float("inf"), -float("inf")):
            r = rows(torch.full((3,), 0.9))
            r[:, col] = bad
            parts.append(r)
    if nc > 1:                                                 # class scores: max below 1, tied, product rounds
        r = rows(0.5 + 0.5 * torch.rand(300, generator=g))
        r[:, 6:] = torch.rand(300, nc, generator=g)
        r[:150, 6] = r[:150, 6 + nc - 1] = r[:150, 6:].max(1).values
        parts.append(r)
    out = torch.cat(parts, 0)
    return out[torch.randperm(len(out), generator=g)].contiguous()


def check_postprocess_equals_per_image(io, conf_thres, nms_thres, cap, min_wh=2.0):
    """nms.detect_postprocess (device-side selection + segmented NMS) == the per-image pipeline (nms_filter -> stable
    top-cap by confidence -> rows back in input order -> r_nms), image by image, bit for bit: the selection is exactly
    the top-cap candidates and the kept boxes are identical.  io [B, P, 7] CUDA.  Returns each image's candidate
    confidences (the filter's survivors, input order)."""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.nms import detect_postprocess, nms_filter
    res = detect_postprocess(io, conf_thres, nms_thres, cap)
    confs = []
    for b in range(io.shape[0]):
        cand = nms_filter(io[b].clone(), conf_thres, min_wh)             # [n, 8] in input order
        confs.append(cand[:, 5])
        top = torch.sort(torch.argsort(cand[:, 5], descending=True, stable=True)[:cap]).values
        want_sel = cand[top][:, :6].contiguous()
        n = int(res["counts"][b])
        assert n == len(want_sel), (b, n, len(want_sel))
        assert torch.equal(res["dets"][b, :n], want_sel), b
        want = want_sel[pkg.r_nms(want_sel, nms_thres)] if len(want_sel) else want_sel
        got = res["dets"][b][res["keep"][b, :int(res["num_keep"][b])]]
        assert got.shape == want.shape, (b, got.shape, want.shape)
        assert torch.equal(got, want), b
    assert res["dets"].shape == (io.shape[0], cap, 6) and res["keep"].shape == (io.shape[0], cap)
    return confs


def init_darknet_weights(model, seed=0):
    """Deterministic non-trivial parameters for a (reference or our) Darknet: He-scaled conv weights, randomised BN
    affine + running statistics and PReLU slopes (defaults mu=0, var=1, slope=0.1 would hide folding bugs,
    SURVEY.md 8d config 5).  Same CPU generator sequence on both sides -> identical weights by state_dict order."""
    g = torch.Generator().manual_seed(seed)
    sd = model.state_dict()
    with torch.no_grad():
        for name, t in sd.items():
            if not t.is_floating_point():
                continue
            shp = tuple(t.shape)
            if name.endswith("Conv2d.weight"):
                fan_in = shp[1] * shp[2] * shp[3]
                v = torch.randn(shp, generator=g) * (0.9 / fan_in) ** 0.5
            elif name.endswith("Conv2d.bias"):
                v = torch.randn(shp, generator=g) * 0.5
            elif name.endswith("BatchNorm2d.weight"):
                v = 0.6 + 0.8 * torch.rand(shp, generator=g)
            elif name.endswith("BatchNorm2d.bias"):
                v = 0.2 * torch.randn(shp, generator=g)
            elif name.endswith("running_mean"):
                v = 0.2 * torch.randn(shp, generator=g)
            elif name.endswith("running_var"):
                v = 0.5 + torch.rand(shp, generator=g)
            elif name.endswith("activation.weight"):
                v = 0.05 + 0.25 * torch.rand(shp, generator=g)
            else:
                v = torch.randn(shp, generator=g) * 0.1
            t.copy_(v.to(t.device))
    return model


SMALL_ANCHORS = "ara 900, 3000, 9000 / 5.0 / -45, 45"   # 6 anchors: one area x 2 angles per scale (same angle set on every scale, as the reference loss assumes)


def cfg_conv(f, k, s=1, bn=1, act="leaky"):
    """one [convolutional] section of a Darknet cfg"""
    return "[convolutional]\n%sfilters=%d\nsize=%d\nstride=%d\npad=1\nactivation=%s\n\n" % (
        "batch_normalize=1\n" if bn else "", f, k, s, act)


def mini_cfg(width=64, height=48):
    """A 19-block graph with every structural feature of cfg/yolov3.cfg (stride-2 convs, shortcuts, a route alias, an
    upsample, a 2-source concat whose second source also feeds a stride-2 conv, two YOLO heads) but only 13 convs, so
    that bf16 noise does not swamp a wiring check.  Reference 'ara' anchor grammar."""
    conv = cfg_conv
    def yolo(lo, hi):
        return "[yolo]\nmask = %d-%d\nanchors = %s\nclasses=1\nnum=6\n\n" % (lo, hi, SMALL_ANCHORS)
    s = "[net]\nwidth=%d\nheight=%d\nchannels=3\n\n" % (width, height)
    s += conv(32, 3) + conv(64, 3, 2) + conv(32, 1) + conv(64, 3) + "[shortcut]\nfrom=-3\nactivation=linear\n\n"
    s += conv(128, 3, 2) + conv(64, 1) + conv(128, 3) + "[shortcut]\nfrom=-3\nactivation=linear\n\n"
    s += conv(64, 1) + conv(21, 1, bn=0, act="linear") + yolo(3, 5)
    s += "[route]\nlayers = -3\n\n" + conv(32, 1) + "[upsample]\nstride=2\n\n[route]\nlayers = -1, 4\n\n"
    s += conv(64, 3) + conv(21, 1, bn=0, act="linear") + yolo(0, 2)
    return s


def wgrad_plan(ksize, cin_pad, cout_pad, batch, h, w, sms, segmented=False):
    """Python mirror of the launch heuristic of ryolo_conv_wgrad and (segmented=True) ryolo_px_wgrad (csrc/wgrad.cu):
    tile width bn, taps per CTA tg, split count; `updates` = wgmma k16 accumulations per split, the length of one
    accumulator chain of ryolo_conv_wgrad (ryolo_px_wgrad restarts it every 32)"""
    np_ = batch * (h + 2) * (w + 2)
    taps = ksize * ksize
    regs = 128 if segmented else 256
    if segmented:
        bn = 128 if cin_pad % 128 == 0 else 64
    else:
        bn = 256 if cin_pad >= 192 else cin_pad
    m_tiles = -(-cout_pad // 128)
    n_tiles = -(-cin_pad // bn)
    ksteps = -(-np_ // 64)
    tg = 1
    if bn <= 128:
        tg = 3 if taps == 9 else (2 if taps == 4 else 1)
    if tg * bn > regs:
        tg = 1
    tiles = (taps // tg) * m_tiles * n_tiles
    ksplit, best = 1, 0.0
    for waves in range(1, 5):
        ks = max(1, waves * sms // tiles)
        ctas = tiles * ks
        eff = ctas / (-(-ctas // sms) * sms)
        if eff > best + 1e-9:
            best, ksplit = eff, ks
        if eff >= 0.9:
            break
    max_split = -(-ksteps // 16)
    ksplit = max(1, min(ksplit, max_split))
    per_split = -(-ksteps // ksplit)
    ksplit = -(-ksteps // per_split)
    last = ksteps - (ksplit - 1) * per_split
    return dict(bn=bn, tg=tg, tiles=tiles, ksteps=ksteps, ksplit=ksplit, per_split=per_split, last=last,
                short_last=last < per_split, n_add=-(-ksteps * 64 // 16) + ksplit, updates=4 * per_split)
