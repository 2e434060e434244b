"""ap_per_class (reference utils/utils.py:200-286) restated in numpy with the tie rule of the device code: rows are
ordered by a STABLE sort on confidence, descending.  On tie-free statistics it is the reference's function
(test_ap_cpu.py checks it against tests/golden/ap_golden.npz bit for bit); the GPU tests compare Evaluator.compute
with it."""
import numpy as np


def ap_per_class(tp, conf, pred_cls, target_cls):
    order = np.argsort(-np.asarray(conf), kind="stable")
    tp, pred_cls = np.asarray(tp, np.float64)[order], np.asarray(pred_cls)[order]
    target_cls = np.asarray(target_cls)
    classes = np.unique(target_cls)
    p, r, ap = [], [], []
    for c in classes:
        sel = pred_cls == c
        n_gt, n_p = (target_cls == c).sum(), sel.sum()
        if n_p == 0:
            p.append(0.0), r.append(0.0), ap.append(0.0)
            continue
        tpc = np.cumsum(tp[sel])
        fpc = np.cumsum(1 - tp[sel])
        recall = tpc / (n_gt + 1e-16)
        precision = tpc / (tpc + fpc)
        r.append(recall[-1]), p.append(precision[-1])
        mrec = np.concatenate(([0.0], recall, [1.0]))
        env = np.maximum.accumulate(np.concatenate(([0.0], precision, [0.0]))[::-1])[::-1]
        i = np.flatnonzero(mrec[1:] != mrec[:-1])
        ap.append(np.sum((mrec[i + 1] - mrec[i]) * env[i + 1]))
    p, r, ap = np.array(p), np.array(r), np.array(ap)
    return p, r, ap, 2 * p * r / (p + r + 1e-16), classes.astype(np.int32)
