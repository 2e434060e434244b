"""csrc/ap.cuh (the per-class arithmetic of ryolo_ap_per_class) built on the host with g++, against the reference's own
ap_per_class (tests/golden/ap_golden.npz, tests/golden/make_golden_ap.py): p, r and f1 bit for bit, AP within 1e-12
relative (the reference's np.sum adds pairwise, the header in row order).  Also: the numpy restatement the GPU tests
use (tests/ap_numpy.py) is the reference on tie-free statistics, and with tied confidences the header follows its
stable order."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from ap_numpy import ap_per_class as ap_stable
from helpers import GOLDEN, REPO

CASES = ("multi", "all_correct", "none_correct", "one_row", "one_row_wrong", "large")

SRC = r'''
#include "ap.cuh"
extern "C" void ap_stats(const int* tp_pos, int ntp, long long n_p, long long n_gt, double* env, double* out) {
  const ryolo::ApClass s = ryolo::ap_class_stats(tp_pos, 0, ntp, n_p, n_gt, env);
  out[0] = s.p; out[1] = s.r; out[2] = s.ap; out[3] = s.f1;
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("ap")
    (d / "ap.cpp").write_text(SRC)
    so = d / "libap.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(REPO, "rotate-yolov3_b200", "csrc"),
                    "-o", str(so), str(d / "ap.cpp")], check=True)
    return ctypes.CDLL(str(so))


def header_ap(lib, tp, conf, pred_cls, target_cls):
    """ryolo_ap_per_class's order (stable by confidence, descending) and per-class walk, with the header's arithmetic"""
    order = np.argsort(-conf, kind="stable")
    tp, pred_cls = np.asarray(tp)[order], pred_cls[order]
    classes = np.unique(target_cls)
    res = np.zeros((len(classes), 4))
    for k, c in enumerate(classes):
        sel = pred_cls == c
        pos = np.ascontiguousarray(np.flatnonzero(tp[sel] != 0), dtype=np.int32)
        env = np.zeros(max(len(pos), 1))
        out = np.zeros(4)
        lib.ap_stats(pos.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(pos)), ctypes.c_longlong(int(sel.sum())),
                     ctypes.c_longlong(int((target_cls == c).sum())), env.ctypes.data_as(ctypes.c_void_p),
                     out.ctypes.data_as(ctypes.c_void_p))
        res[k] = out
    return res[:, 0], res[:, 1], res[:, 2], res[:, 3], classes.astype(np.int32)


def _golden(case):
    g = np.load(os.path.join(GOLDEN, "ap_golden.npz"))
    ins = [g["%s_%s" % (case, k)] for k in ("tp", "conf", "pred_cls", "target_cls")]
    outs = [g["%s_%s" % (case, k)] for k in ("p", "r", "ap", "f1", "ap_class")]
    return ins, outs


def check_close(got, want):
    p, r, ap, f1, cls = got
    wp, wr, wap, wf1, wcls = want
    assert np.array_equal(cls, wcls)
    for a, b in ((p, wp), (r, wr), (f1, wf1)):
        assert np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))
    assert np.all(np.abs(ap - wap) <= 1e-12 * np.abs(wap)), np.abs(ap - wap).max()


@pytest.mark.parametrize("case", CASES)
def test_header_reproduces_reference_golden(lib, case):
    ins, want = _golden(case)
    check_close(header_ap(lib, *ins), want)


@pytest.mark.parametrize("case", CASES)
def test_numpy_restatement_is_the_reference(case):
    ins, want = _golden(case)
    got = ap_stable(*ins)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_golden_covers_the_cases():
    _, (p, r, ap, f1, cls) = _golden("multi")
    ins, _ = _golden("multi")
    assert 3 in ins[2] and 3 not in ins[3]          # a predicted class without targets
    assert 2 in ins[3] and 2 not in ins[2]          # a target class without predictions
    assert ap[list(cls).index(2)] == 0 and p[list(cls).index(2)] == 0
    assert len(_golden("one_row")[0][0]) == 1
    assert _golden("all_correct")[0][0].all() and not _golden("none_correct")[0][0].any()


def test_ties_follow_the_stable_order(lib):
    """confidences on a coarse grid: every class has long runs of ties, and the order inside a run changes the AP"""
    rng = np.random.default_rng(11)
    n = 3000
    conf = (rng.integers(1, 40, n) / 40.0).astype(np.float32)
    pred_cls = rng.integers(0, 3, n).astype(np.float32)
    tp = (rng.random(n) < 0.3).astype(np.float64)
    target_cls = np.repeat(np.arange(4, dtype=np.float32), [400, 350, 500, 9])
    got = header_ap(lib, tp, conf, pred_cls, target_cls)
    check_close(got, ap_stable(tp, conf, pred_cls, target_cls))
    rev = np.arange(n)[::-1]        # the same rows, ties in the opposite order
    other = ap_stable(tp[rev], conf[rev], pred_cls[rev], target_cls)
    assert not np.array_equal(other[2], got[2])
