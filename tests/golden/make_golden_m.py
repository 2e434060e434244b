#!/usr/bin/env python
"""Golden fixtures of the reference's multi-branch dilated graph (cfg/yolov3-m.cfg, cfg/HRSC/yolov3-m.cfg,
cfg/HRSC+/yolov3_512_matrix.cfg): the REFERENCE Darknet (model/models.py: [d-convolutional] :68-77, weight_from
:255-265) run here on CPU in fp32, weights from helpers.init_darknet_weights.

The reference parser cannot read these cfgs as shipped.  yolov3-m's anchor line lacks the `ara` token (SURVEY.md D3),
so the reference is given a copy with `ara` inserted, the same fix as for cfg/yolov3.cfg.  The matrix cfg names an
anchor file the reference does not ship, so its copy gets MATRIX_ANCHORS (stored below; the tests supply the same line).

    darknet_m_golden.npz
      tree:<cfg>       repr() of the reference's module_list
      state:<cfg>      JSON [[state_dict key, shape], ...]
      n_params:<cfg>   parameter count
      weights_sha256   sha256 of the reference's save_weights file of yolov3-m.cfg with weights seed SEEDS["eval_w"]
      eval_*           yolov3-m.cfg, eval, batch 1 at 416 x 416: samples of the 16 heads (with each head's |max|) and
                       of the decoded rows

Inputs and sample positions are regenerated from seeds by tests/test_dilated_gpu.py.  Not run by the test-suite (the
GPU box has no reference tree).  Re-run: python tests/golden/make_golden_m.py"""
import hashlib
import json
import os
import re
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(REPO, "tests"))

CFGS = ["cfg/yolov3-m.cfg", "cfg/HRSC/yolov3-m.cfg", "cfg/HRSC+/yolov3_512_matrix.cfg"]
MATRIX_ANCHORS = "ara 792, 2061, 3870, 6353, 9623, 15803 / 4.18, 6.48, 8.71 / -75, -60, -45, -30, -15, 0, 15, 30, 45, 60, 75, 90"
SEEDS = dict(eval_w=610, eval_x=6100, train_w=611, train_x=6110)
ARCS = ("default", "Fdefault")
HYP = {"giou": 0.1, "cls": 27.76, "cls_pw": 1.0, "obj": 20.35, "obj_pw": 1.0, "iou_t": 0.5, "ang_t": 3.1415926 / 12,
       "reg": 1.0, "context_factor": 1.0, "fl_gamma": 1.5}


def train_targets():
    """[image, class, x, y, w, h, theta] of the training fixture: sizes near the area-792 / ratio-4.18 anchors (57.5 x
    13.8 px on the 160 x 128 image), so that every target has a matching anchor"""
    t = torch.tensor([[0, 0, 0.30, 0.40, 57.5 / 160, 13.8 / 128, 0.5],
                      [0, 0, 0.70, 0.60, 60.0 / 160, 14.5 / 128, -0.9],
                      [1, 0, 0.50, 0.50, 55.0 / 160, 13.0 / 128, 1.2],
                      [1, 0, 0.20, 0.80, 58.0 / 160, 14.0 / 128, -0.3]])
    return t


def reference_readable(text):
    """the cfg text with every anchor line in the `ara` grammar the reference parser reads"""
    def fix(m):
        val = m.group(2).strip()
        if "," not in val:                       # an anchor file path (the matrix cfg)
            val = MATRIX_ANCHORS
        elif "ara" not in val:
            val = "ara " + val
        return m.group(1) + val
    return re.sub(r"^(anchors\s*=)(.*)$", fix, text, flags=re.M)


def sample_idx(numel, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, numel, (n,), generator=g)


def main():
    import make_golden as mg
    import helpers
    _, _, rmodels, _ = mg.import_reference()
    from model.model_utils import save_weights
    torch.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    sav = {"seeds": np.array(json.dumps(SEEDS).encode()), "matrix_anchors": np.array(MATRIX_ANCHORS.encode())}
    tmp = tempfile.mkdtemp()
    paths = {}
    for c in CFGS:
        paths[c] = os.path.join(tmp, c.replace("/", "_"))
        with open(c) as f, open(paths[c], "w") as g:
            g.write(reference_readable(f.read()))
        m = rmodels.Darknet(paths[c], {"context_factor": 1.0}, arc="default")
        sav["tree:" + c] = np.array(repr(m.module_list).encode())
        sav["state:" + c] = np.array(json.dumps([[k, list(v.shape)] for k, v in m.state_dict().items()]).encode())
        sav["n_params:" + c] = sum(p.numel() for p in m.parameters())
        print(c, sav["n_params:" + c])

    model = rmodels.Darknet(paths[CFGS[0]], {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=SEEDS["eval_w"])
    wpath = os.path.join(tmp, "m.weights")
    save_weights(model, wpath)
    with open(wpath, "rb") as f:
        sav["weights_sha256"] = np.array(hashlib.sha256(f.read()).hexdigest().encode())
    sav["weights_bytes"] = os.path.getsize(wpath)

    model.eval()
    x = torch.rand(1, 3, 416, 416, generator=torch.Generator().manual_seed(SEEDS["eval_x"]))
    with torch.no_grad():
        io, ps = model(x)
    for k, p in enumerate(ps):
        flat = p.reshape(-1)
        sav["eval_p%d" % k] = flat[sample_idx(flat.numel(), 2048, 100 + k)].numpy()
        sav["eval_p%d_absmax" % k] = float(flat.abs().max())
        sav["eval_p%d_shape" % k] = np.array(p.shape)
    sav["eval_io_rows"] = io[0, sample_idx(io.shape[1], 4000, 110)].numpy()
    sav["eval_io_shape"] = np.array(io.shape)
    print("eval:", tuple(io.shape), len(ps), [round(sav["eval_p%d_absmax" % k], 3) for k in range(len(ps))])
    # ---- training step at 160 x 128, batch 2: compute_loss (default and Fdefault arcs) and every gradient ----
    import model.loss as rloss
    torch.Tensor.cuda = lambda self, *a, **k: self          # loss.py:197 hard-codes .cuda()
    for arc in ARCS:
        model = rmodels.Darknet(paths[CFGS[0]], HYP, arc=arc)
        helpers.init_darknet_weights(model, seed=SEEDS["train_w"])
        model.hyp, model.nc, model.arc = HYP, 1, arc
        model.train()
        x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(SEEDS["train_x"]))
        ps = model(x)
        loss, items = rloss.compute_loss(ps, train_targets(), model, HYP)
        loss.backward()
        sav[arc + "_loss"], sav[arc + "_items"] = float(loss), items.detach().numpy()
        names, has, norms, samples = [], [], [], []
        for j, (name, prm) in enumerate(model.named_parameters()):
            names.append(name)
            has.append(prm.grad is not None)
            if prm.grad is None:
                norms.append(np.nan)
                samples.append(np.zeros(0, dtype=np.float32))
                continue
            gflat = prm.grad.reshape(-1)
            samples.append(gflat[sample_idx(gflat.numel(), 256, 1000 + j)].numpy())
            norms.append(float(gflat.double().norm()))
        sav[arc + "_names"], sav[arc + "_has_grad"] = np.array(names), np.array(has)
        sav[arc + "_norms"], sav[arc + "_samples"] = np.array(norms), np.array(samples, dtype=object)
        for k in (0, 4, 12, 111):
            flat = ps[k].detach().reshape(-1) if k < len(ps) else None
            if flat is not None:
                sav[arc + "_p%d" % k] = flat[sample_idx(flat.numel(), 2048, 200 + k)].numpy()
                sav[arc + "_p%d_absmax" % k] = float(flat.abs().max())
        print("train %s: loss %.5f items %s, %d parameters, %d without gradient" % (
            arc, float(loss), items.numpy(), len(names), len(names) - sum(has)))

    out = os.path.join(HERE, "darknet_m_golden.npz")
    np.savez_compressed(out, **sav)
    print("wrote", out, os.path.getsize(out))


if __name__ == "__main__":
    main()
