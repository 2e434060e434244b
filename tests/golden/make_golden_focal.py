#!/usr/bin/env python
"""Generates tests/golden/loss_focal_golden.npz by RUNNING THE REFERENCE's compute_loss (model/loss.py:266-367) with a
focal arc ('Fdefault': FocalLoss around every criterion, :284-286) on the CPU.  Not run by the test-suite.  Re-run:
`python tests/golden/make_golden_focal.py` (the reference sources at /root/reference, imported with the stubs and the
.cuda() shim of make_golden.py section 9).

Outputs only: the inputs are rebuilt by tests/focal_cases.py from loss_golden.npz and seeds.
  a_g{gamma}_pw{obj_pw}_*  the heads and targets of loss_golden.npz, gamma in {0.5, 2}, obj_pw in {1, 2}: loss, items,
                           the gradient of every head
  b_g{gamma}_*             the same heads without targets
  c_g{gamma}_*             extreme objectness logits (focal_cases.extreme_heads) with the targets
  d_*                      the section-7 Darknet-53 model (160 x 128, batch 4) trained with the Fdefault loss: loss,
                           items, gradient samples and norms of every parameter
nc = 1 throughout: the reference's nc > 1 branch feeds BCE an [nb, nc + 1] input against an [nb, nc] target and raises."""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, REPO)

import focal_cases as FC  # noqa: E402
import helpers  # noqa: E402
from make_golden import import_reference  # noqa: E402


def main():
    torch.set_num_threads(8)
    _, _, rmodels, _ = import_reference()
    import model.loss as rloss
    torch.Tensor.cuda = lambda self, *a, **k: self          # loss.py:197 hard-codes .cuda()
    from rotate_yolov3_b200 import cfgs
    text = cfgs.yolov3_cfg(width=160, height=128, classes=1, anchors=helpers.SMALL_ANCHORS, n_anchors=6)
    with tempfile.NamedTemporaryFile("w", suffix=".cfg", delete=False) as f:
        f.write(text)
        cfg_path = f.name
    model = rmodels.Darknet(cfg_path, {"context_factor": 1.0}, arc="Fdefault")
    helpers.init_darknet_weights(model, seed=321)
    model.train()
    x, tg_d, hyp_d = FC.darknet_case()
    ps = model(x)                                      # sets ng / anchor_vec of the YOLO layers (also for a-c)
    model.nc, model.arc = 1, "Fdefault"
    heads, tg, hyp0 = FC.base_inputs()
    sav = {}

    def run(tag, hs, targets, hyp):
        model.hyp = hyp
        pl = [h.detach().clone().requires_grad_(True) for h in hs]
        loss, items = rloss.compute_loss(pl, targets.clone(), model, hyp)
        loss.backward()
        sav[tag + "_loss"], sav[tag + "_items"] = loss.detach().numpy(), items.numpy()
        for k, p in enumerate(pl):
            sav[tag + "_dp%d" % k] = p.grad.numpy()
        print(tag, items.numpy())

    for gm in FC.GAMMAS:
        for pw in FC.OBJ_PWS:
            run("a_g%g_pw%g" % (gm, pw), heads, tg, FC.focal_hyp(hyp0, gm, pw))
        run("b_g%g" % gm, heads, torch.zeros(0, 7), FC.focal_hyp(hyp0, gm, hyp0["obj_pw"]))
        run("c_g%g" % gm, FC.extreme_heads(heads), tg, FC.focal_hyp(hyp0, gm, hyp0["obj_pw"]))

    # (d) the whole network trained with the focal loss
    model.hyp = hyp_d
    loss, items = rloss.compute_loss(ps, tg_d.clone(), model, hyp_d)
    loss.backward()
    sav["d_loss"], sav["d_items"] = loss.detach().numpy(), items.numpy()
    names, norms, samples, sample_idx = [], [], [], []
    gi = torch.Generator().manual_seed(12)
    for name, prm in model.named_parameters():
        gflat = prm.grad.reshape(-1)
        idx = torch.randint(0, gflat.numel(), (min(256, gflat.numel()),), generator=gi)
        names.append(name)
        norms.append(float(gflat.norm()))
        sample_idx.append(idx.numpy())
        samples.append(gflat[idx].numpy())
    sav["d_names"] = np.array(names)
    sav["d_norms"] = np.array(norms)
    sav["d_sample_idx"] = np.array(sample_idx, dtype=object)
    sav["d_samples"] = np.array(samples, dtype=object)
    np.savez_compressed(os.path.join(HERE, "loss_focal_golden.npz"), **sav)
    print("d", items.numpy(), "%d params, grad norm range %.3e .. %.3e" % (len(names), min(norms), max(norms)))


if __name__ == "__main__":
    main()
