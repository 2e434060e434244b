#!/usr/bin/env python
"""Golden fixture of the mAP statistics: the REFERENCE's own ``ap_per_class`` / ``compute_ap`` (utils/utils.py:200-286),
run here on the CPU over seeded statistics shaped like test.py's (correct, conf, pred_cls, target_cls).

    ap_golden.npz, per case <c>:
        <c>_tp, <c>_conf, <c>_pred_cls, <c>_target_cls     the inputs (tp as test.py concatenates it: float64 0 / 1)
        <c>_p, <c>_r, <c>_ap, <c>_f1, <c>_ap_class         the reference's outputs

Cases: several classes with a predicted class that has no targets and a target class with no predictions, all-correct,
none-correct, one row, and a large multi-class set whose AP sums run past numpy's pairwise-summation block.  Confidences
are distinct within a case, so the reference's unstable argsort has one answer.
Not run by the test-suite (the GPU box has no reference checkout).  Re-run: python tests/golden/make_golden_ap.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def stats(seed, n, pred_classes, target_counts, tp_rate):
    """n rows with distinct float32 confidences, classes drawn from pred_classes; per class at most target_counts[c]
    rows are correct (each target is claimed once), chosen at random with probability tp_rate"""
    rng = np.random.default_rng(seed)
    conf = rng.permutation(np.linspace(0.001, 0.999, n, dtype=np.float32))
    pred_cls = rng.choice(np.asarray(pred_classes, np.float32), n)
    tp = np.zeros(n)
    for c, k in target_counts.items():
        rows = np.flatnonzero((pred_cls == c) & (rng.random(n) < tp_rate))
        tp[rows[:k]] = 1.0
    target_cls = np.repeat(np.asarray(list(target_counts), np.float32), list(target_counts.values()))
    return tp, conf, pred_cls, rng.permutation(target_cls)


CASES = {
    # classes 0, 1 and 3 predicted, 0, 1 and 2 in the targets: 3 has no targets, 2 no predictions
    "multi": stats(1, 300, [0, 1, 3], {0: 40, 1: 25, 2: 7}, 0.4),
    "all_correct": (np.ones(20), *stats(2, 20, [0], {0: 25}, 1.0)[1:]),
    "none_correct": stats(3, 15, [0], {0: 4}, 0.0),
    "one_row": stats(4, 1, [0], {0: 1}, 1.0),
    "one_row_wrong": stats(5, 1, [0], {0: 3}, 0.0),
    "large": stats(6, 20000, [0, 1, 2, 4], {0: 900, 1: 350, 2: 1200, 3: 60, 4: 5}, 0.5),
}


def main():
    import make_golden as mg
    ru = mg.import_reference()[0]
    out = {}
    for name, (tp, conf, pred_cls, target_cls) in CASES.items():
        p, r, ap, f1, ap_class = ru.ap_per_class(tp.copy(), conf.copy(), pred_cls.copy(), target_cls.copy())
        for key, val in (("tp", tp), ("conf", conf), ("pred_cls", pred_cls), ("target_cls", target_cls), ("p", p),
                         ("r", r), ("ap", ap), ("f1", f1), ("ap_class", ap_class)):
            out["%s_%s" % (name, key)] = np.asarray(val)
        print("%-14s rows %5d  classes %s  ap %s" % (name, len(tp), ap_class.tolist(), np.round(ap, 4).tolist()))
    np.savez_compressed(os.path.join(HERE, "ap_golden.npz"), **out)


if __name__ == "__main__":
    main()
