"""TEST INFRASTRUCTURE: the letterbox fixture's cases and the numpy restatements of the letterbox step
(rotate-yolov3_b200/preprocess.py) that test_letterbox_cpu.py and test_letterbox_gpu.py check against, and
test_augment_cpu.py reuses for the pre-resize."""
import numpy as np


def source(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def net_input(lb, dtype):
    x = np.ascontiguousarray(lb[:, :, ::-1].transpose(2, 0, 1), dtype=dtype)
    x /= 255.0
    return x


def letterbox_case(g, name):
    k = "case_%s_" % name
    ns = g[k + "new_shape"]
    new_shape = int(ns[0]) if str(g[k + "mode"]) == "square" else (int(ns[0]), int(ns[1]))
    h, w = (int(v) for v in g[k + "src"])
    return source(int(g[k + "seed"]), h, w), new_shape, str(g[k + "mode"]), k


def resize_np(img, dst_hw):
    """what ryolo_letterbox computes for the resized region, restated in numpy from resample_tables"""
    import rotate_yolov3_b200.preprocess as pp
    kind, (kx, ky), (xs, xn, xw), (ys, yn, yw) = pp.resample_tables(img.shape[:2], dst_hw)
    sh, sw = img.shape[:2]
    dh, dw = dst_hw
    out = np.zeros((dh, dw, 3), np.uint8)
    src = img.astype(np.int64)
    if kind == pp.AREA_INT:
        for y in range(dh):
            blk = src[ys[y]:ys[y] + ky].reshape(ky, dw, kx, 3).sum((0, 2))
            if kx == 2 and ky == 2:
                out[y] = (blk + 2) >> 2
            else:
                out[y] = np.clip(np.rint(blk.astype(np.float32) * (np.float32(1) / np.float32(kx * ky))), 0, 255)
        return out
    if kind == pp.LINEAR:
        x1 = np.minimum(np.array(xs) + 1, sw - 1)
        a0 = np.array([w[0] for w in xw])[:, None]
        a1 = np.array([w[1] for w in xw])[:, None]
        for y in range(dh):
            r0, r1 = ys[y], min(ys[y] + 1, sh - 1)
            b0, b1 = yw[y]
            h0 = src[r0, xs] * a0 + src[r0, x1] * a1
            h1 = src[r1, xs] * a0 + src[r1, x1] * a1
            out[y] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2
        return out
    srcf = img.astype(np.float32)
    xs, xn = np.array(xs), np.array(xn)
    wpad = np.zeros((dw, xn.max()), np.float32)                 # zero weights past a pixel's taps add exactly nothing
    for x in range(dw):
        wpad[x, :xn[x]] = xw[x]
    for y in range(dh):
        acc = np.zeros((dw, 3), np.float32)
        for j in range(yn[y]):
            row = srcf[ys[y] + j]
            buf = np.zeros((dw, 3), np.float32)
            for i in range(xn.max()):
                buf = buf + row[np.minimum(xs + i, sw - 1)] * wpad[:, i:i + 1]
            acc = acc + np.float32(yw[y][j]) * buf
        out[y] = np.clip(np.rint(acc), 0, 255)
    return out
