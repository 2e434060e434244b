"""The streams cv2 never writes (tests/jpeg_syntax_cases.py, checked first by the host build in
test_jpeg_syntax_cpu.py) through decode_images on the device, mixed into one call with the cv2-written matrix: every
image equals cv2.imread of the same file, the range cases go to the host, the matrix stays on the device.  Prints the
cv2 build's JPEG / SIMD lines and the CPU's avx2 flag, since which IDCT cv2 runs depends on them."""
import cv2
import numpy as np
import pytest
import torch

import jpeg_syntax_cases as cases
from jpeg_cases import matrix

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _host_simd():
    lines = [ln.strip() for ln in cv2.getBuildInformation().splitlines() if "JPEG" in ln or "SIMD" in ln]
    try:
        avx2 = " avx2 " in " " + open("/proc/cpuinfo").read().replace("\n", " ") + " "
    except OSError:
        avx2 = None
    return lines, avx2


def _imread(tmp_path, blobs):
    out = []
    for i, b in enumerate(blobs):
        p = tmp_path / ("%d.jpg" % i)
        p.write_bytes(b)
        out.append(cv2.imread(str(p)))
    return out


@pytest.mark.parametrize("chunk", [128, 3])
def test_syntax_cases_with_matrix_in_one_call(tmp_path, chunk):
    from rotate_yolov3_b200 import decode_images
    lines, avx2 = _host_simd()
    print("cv2:", lines, "avx2:", avx2)
    syn = [c for c in cases.all_cases()]
    nat = [(n, b, "device") for n, b in matrix()]
    items = syn + nat
    want = _imread(tmp_path, [b for _, b, _ in items])
    keep = [(it, w) for it, w in zip(items, want) if w is not None]
    assert len(keep) == len(items), [it[0] for it, w in zip(items, want) if w is None]
    imgs, routes = decode_images([it[1] for it, _ in keep], device=DEV, chunk_bytes=chunk)
    torch.cuda.synchronize()
    bad = []
    for ((name, _, expect), w), img, route in zip(keep, imgs, routes):
        got = img.cpu().numpy()
        if got.shape != w.shape or (got != w).any():
            bad.append((name, "differs from cv2.imread", route))
        if expect == "device" and route != "device":
            bad.append((name, route))
        if expect == "range" and "outside the IDCT" not in route:
            bad.append((name, route))
        if expect == "host" and route == "device":
            bad.append((name, route))
    assert not bad, bad
