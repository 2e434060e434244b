"""TEST INFRASTRUCTURE: the literal, indexed restatement of the reference's ``build_targets`` / ``compute_loss``
(model/loss.py:161-258, 266-367; statement order and names follow the reference so that the two can be read side by
side).  It is the CHECKER of the sync-free masked formulation in rotate-yolov3_b200/loss.py and is itself pinned to the
reference's outputs by tests/golden/loss_golden.npz.  Not part of the product package (VERDICT r1, copy-paste findings)."""
import math

import torch
import torch.nn as nn

from rotate_yolov3_b200.loss import wh_iou


def build_targets(model, targets, hyp):
    """targets [nt, 7] = (image, class, x, y, w, h, theta), normalised xywh.  Returns tcls, tbox, indices, av per YOLO
    layer (model/loss.py:161-258).  Like the reference, the context factor is applied to ``targets`` in place once per
    YOLO layer (harmless for the shipped context_factor = 1.0)."""
    nt = len(targets)
    tcls, tbox, indices, av, square_ious = [], [], [], [], []
    dev = targets.device
    all_ious = None
    na = 0
    t_gwha = None
    anchor_vec = None
    for i in model.yolo_layers:
        layer = model.module_list[i]
        ng, anchor_vec = layer.ng.to(dev), layer.anchor_vec.to(dev)
        targets[:, 4] += targets[:, 5] * (hyp["context_factor"] - 1)
        targets[:, 5] *= hyp["context_factor"]
        t, a = targets, []
        gwha = t[:, 4:7].clone()
        gwha[:, :-1] *= ng
        if nt:
            all_ious = torch.stack([wh_iou(x, gwha[:, :-1]) for x in anchor_vec[:, :-1]], 0)   # [na, nt]
            na = len(anchor_vec)
            a = torch.arange(na, device=dev).view((-1, 1)).repeat([1, nt]).view(-1)
            t = targets.repeat([na, 1])
            gwha = gwha.repeat([na, 1])
            square_ious.append(all_ious.view(-1))
        b, c = t[:, :2].long().t()
        gxy = t[:, 2:4] * ng
        gi, gj = gxy.long().t()
        indices.append([b, a, gj, gi])
        gxy = gxy - gxy.floor()
        t_gwha = gwha.clone()
        tbox.append(torch.cat((gxy, gwha), 1))
        av.append(anchor_vec[a] if nt else anchor_vec[:0])
        tcls.append(c)
    if nt:
        nl = len(model.yolo_layers)
        angle_offset = (t_gwha[:, -1] - anchor_vec[:, -1].view((-1, 1)).repeat([1, nt]).view(-1)).abs()
        big = angle_offset > 0.5 * math.pi
        angle_offset[big] = math.pi - angle_offset[big]
        j_a = angle_offset < model.hyp["ang_t"]
        j = [(sq > model.hyp["iou_t"]) & j_a for sq in square_ious]
        gt_j = torch.stack([juu.reshape(all_ious.shape).max(0)[0] for juu in j], 0).t()    # [nt, layers]
        # Host synchronisations are kept to a handful (one per device->host read below): the reference walks the targets
        # in a Python loop with one sync each, which on a GPU costs more than the whole loss arithmetic.
        class_ok = tcls[0].max() <= model.nc
        orphans = (~gt_j.any(1)).nonzero().view(-1).tolist()                                # sync 1
        for gt_id in orphans:       # a GT no anchor of any layer accepted: give it its best-IoU anchor (:235-242)
            gt_ious = torch.cat([sq[gt_id::nt] for sq in square_ious], 0)
            best = torch.where(gt_ious == gt_ious.max(0)[0])[0]
            layer_id = int((best // na)[0])
            best_ang = angle_offset[gt_id::nt].repeat(nl)[best].min(0)[1]
            best = best[best_ang]
            j[layer_id][(best % na) * nt + gt_id] = True
        keep = [m.nonzero().view(-1) for m in j]                                            # syncs 2..nl+1
        assert bool(class_ok), "Target classes exceed model classes"
        assert sum(len(k) for k in keep) >= nt, "something wrong at target building"
        for lid, k in enumerate(keep):
            tbox[lid] = tbox[lid][k]
            tcls[lid] = tcls[lid][k]
            av[lid] = av[lid][k]
            indices[lid] = [indices[lid][q][k] for q in range(4)]
    return tcls, tbox, indices, av


def compute_loss_indexed(p, targets, model, hyp):
    dev = p[0].device
    lcls = torch.zeros(1, device=dev)
    lobj = torch.zeros(1, device=dev)
    lreg = torch.zeros(1, device=dev)
    tcls, tbox, indices, anchor_vecs = build_targets(model, targets, hyp)
    h = model.hyp
    arc = model.arc
    if "default" not in arc or "F" in arc:
        raise NotImplementedError("only arc='default' is restated (the configuration the reference ships)")
    BCEcls = nn.BCEWithLogitsLoss(pos_weight=torch.tensor([h["cls_pw"]], device=dev))
    BCEobj = nn.BCEWithLogitsLoss(pos_weight=torch.tensor([h["obj_pw"]], device=dev))
    SM = nn.SmoothL1Loss(reduction="mean")
    for i, pi in enumerate(p):
        b, a, gj, gi = indices[i]
        tobj = torch.zeros_like(pi[..., 0])
        nb = len(b)
        if nb:
            ps = pi[b, a, gj, gi]
            tobj[b, a, gj, gi] = 1.0
            av = model.module_list[model.yolo_layers[i]].anchor_vec.to(dev)
            pxy = torch.sigmoid(ps[:, 0:2])
            pwh = torch.exp(ps[:, 2:4]).clamp(max=1e3) * av[a][:, :-1]
            pa = torch.atan(ps[:, 4]) + av[a][:, -1]
            liou = (1.0 - wh_iou(tbox[i][:, 2:4], pwh)).mean()
            lreg = lreg + SM(pxy, tbox[i][:, [0, 1]]) + 2 * SM(pa, tbox[i][:, 4]) + liou * h["giou"]
            if model.nc > 1:
                t = torch.zeros_like(ps[:, 6:])
                t[range(nb), tcls[i]] = 1.0
                lcls = lcls + BCEcls(ps[:, 5:], t)     # (reference passes ps[:, 5:] -- obj column included -- vs a [nb, nc] target
                                                      #  only when nc > 1; shapes as in the reference)
        lobj = lobj + BCEobj(pi[..., 5], tobj)         # NoSampler: the whole map (loss.py:24-28, 346-348)
    lobj = lobj * h["obj"]
    lcls = lcls * h["cls"]
    lreg = lreg * h["reg"]
    loss = lobj + lcls + lreg
    return loss, torch.cat((lobj, lcls, lreg, loss)).detach()
