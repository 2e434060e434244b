"""``compute_loss`` / ``build_targets`` with the reference's semantics (model/loss.py:161-258, 266-367; wh_iou
utils/utils.py:346-361), restated device-agnostically (the reference hard-codes ``.cuda()`` at loss.py:197).  This is the
CONSUMER of the training hot path (SURVEY.md 8a row a6): tiny tensors, plain PyTorch on whatever device ``p`` lives on.

Covered: the arcs containing 'default' (separate obj / cls BCE) -- 'default', and with 'F' ('Fdefault', 'Fdefaultpw')
the focal form of model/loss.py:126-146, 284-286 with gamma = hyp['fl_gamma'] -- NoSampler, reject=True target
assignment with the orphan-GT rescue.  Regression loss = SmoothL1(sigmoid xy) + 2 SmoothL1(theta) + giou * mean(1 -
wh_iou): there is no rotated IoU in the reference loss (SURVEY.md D1).  The unified arcs ('uBCE', 'uFBCE', 'uCE',
'uFCE') raise NotImplementedError."""
import ctypes
import math

import torch
import torch.nn as nn


def wh_iou(box1, box2):
    """utils/utils.py:346-361"""
    if box1.shape != box2.shape:
        box2 = box2.t()
        w1, h1 = box1[0], box1[1]
        w2, h2 = box2[0], box2[1]
    else:
        w1, h1 = box1[:, 0], box1[:, 1]
        w2, h2 = box2[:, 0], box2[:, 1]
    inter = torch.min(w1, w2) * torch.min(h1, h2)
    return inter / ((w1 * h1 + 1e-16) + w2 * h2 - inter)


def _targets_masked(model, targets, hyp):
    """The target assignment of build_targets WITHOUT its data-dependent filtering: every (anchor, target) pair keeps its
    row and a boolean mask says which rows the reference would have kept.  All shapes are functions of (na, nt) only, so
    nothing here reads a device value on the host -- on a GPU the indexed formulation costs ~10 host synchronisations
    (each one drains the queue of the 75-layer forward) and leaves the device idle for longer than the loss itself takes.
    Same arithmetic as build_targets (model/loss.py:161-258), including the orphan-GT rescue (:235-242) vectorised over
    the targets."""
    nt = len(targets)
    dev = targets.device
    out = []
    square_ious = []
    anchor_vec = None
    na = 0
    t_gwha = None
    for i in model.yolo_layers:
        layer = model.module_list[i]
        ng, anchor_vec = layer.ng.to(dev), layer.anchor_vec.to(dev)
        targets[:, 4] += targets[:, 5] * (hyp["context_factor"] - 1)
        targets[:, 5] *= hyp["context_factor"]
        gwha = targets[:, 4:7].clone()
        gwha[:, :-1] *= ng
        # wh_iou of every anchor with every target in one shot (same element-wise arithmetic as the reference's
        # per-anchor loop, which on a GPU costs ~8 kernel launches per anchor)
        w1, h1 = anchor_vec[:, 0:1], anchor_vec[:, 1:2]                  # [na, 1]
        w2, h2 = gwha[:, 0].view(1, -1), gwha[:, 1].view(1, -1)          # [1, nt]
        inter = torch.min(w1, w2) * torch.min(h1, h2)
        all_ious = inter / ((w1 * h1 + 1e-16) + w2 * h2 - inter)         # [na, nt]
        na = len(anchor_vec)
        a = torch.arange(na, device=dev).view((-1, 1)).repeat([1, nt]).view(-1)
        t = targets.repeat([na, 1])
        gwha = gwha.repeat([na, 1])
        square_ious.append(all_ious.reshape(-1))
        b, c = t[:, :2].long().t()
        gxy = t[:, 2:4] * ng
        gi, gj = gxy.long().t()
        gxy = gxy - gxy.floor()
        t_gwha = gwha
        out.append(dict(b=b, a=a, gj=gj, gi=gi, tbox=torch.cat((gxy, gwha), 1), av=anchor_vec[a], tcls=c))
    nl = len(model.yolo_layers)
    angle_offset = (t_gwha[:, -1] - anchor_vec[:, -1].view((-1, 1)).repeat([1, nt]).view(-1)).abs()
    angle_offset = torch.where(angle_offset > 0.5 * math.pi, math.pi - angle_offset, angle_offset)
    j_a = angle_offset < model.hyp["ang_t"]
    j = [((sq > model.hyp["iou_t"]) & j_a).view(na, nt) for sq in square_ious]
    gt_any = torch.stack([m.any(0) for m in j], 0).any(0)                      # [nt]: some anchor of some layer accepted
    # orphan rescue: best IoU over all layers' anchors; among ties the smallest angle offset picks the ANCHOR, the first
    # tie picks the LAYER (the reference's `(best // na)[0]` next to `best[best_ang]`)
    G = torch.stack(square_ious, 0).view(nl * na, nt)
    cand = G == G.max(0)[0]
    layer_id = cand.float().argmax(0) // na                                     # argmax returns the FIRST maximum
    ang = angle_offset.view(na, nt).repeat(nl, 1)
    best = torch.where(cand, ang, torch.full_like(ang, float("inf"))).argmin(0)  # first minimum among the candidates
    anchor = best % na
    orphan = ~gt_any
    onehot = torch.arange(na, device=dev).view(-1, 1) == anchor.view(1, -1)     # [na, nt]
    for lid in range(nl):
        m = j[lid] | (onehot & (orphan & (layer_id == lid)).view(1, -1))
        out[lid]["mask"] = m.view(-1)
    return out


# 1.000001 - 1 as the reference's fp32 focal factor sees it (the scalar rounds to the float 1 + 2^-20)
_FOCAL_EPS = 2.0 ** -20


def _focal_gamma(model):
    """the focal exponent of the model's arc: None for the plain arcs, hyp['fl_gamma'] for arcs with 'F' (a missing key
    raises KeyError like model/loss.py:285); arcs without 'default' are not restated"""
    arc = model.arc
    if "default" not in arc:
        raise NotImplementedError("arc %r is not supported: compute_loss restates the arcs containing 'default' "
                                  "('default', 'Fdefault', 'Fdefaultpw'), not the unified 'uBCE' / 'uCE' forms" % (arc,))
    return float(model.hyp["fl_gamma"]) if "F" in arc else None


def _focal(l, gamma):
    """FocalLoss of model/loss.py:126-146 on the element losses l (alpha = 1): l * (1.000001 - exp(-l))^gamma, the base
    written as 2^-20 - expm1(-l) so that it does not cancel for small l; gamma None = the plain loss"""
    if gamma is None:
        return l
    return l * (_FOCAL_EPS - torch.expm1(-l.clamp(min=0.0))) ** gamma


def compute_loss(p, targets, model, hyp):
    """p: list of [B, na, ny, nx, nc+6] raw head tensors (training-mode output of Darknet); returns (loss[1],
    detached (lobj, lcls, lreg, loss)) like model/loss.py:266-367 for the arcs containing 'default' (with 'F': focal).

    The reference selects the matched (anchor, target) rows with data-dependent indexing (build_targets, loss.py:161-258:
    ~350 device-to-host reads per step); this evaluates the same sums over ALL (anchor, target) rows weighted by the 0/1
    assignment mask -- no host synchronisation.  tests/loss_indexed.py holds the literal indexed restatement and
    tests/test_loss.py proves the two equal (value, components, gradients) and pins both to the reference's outputs."""
    if p[0].is_cuda and p[0].dtype == torch.float32:
        return _compute_loss_fused(p, targets, model, hyp)
    if len(targets) == 0:
        return _compute_loss_no_targets(p, model)
    return _compute_loss_masked(p, targets, model, hyp)


def _compute_loss_no_targets(p, model):
    """no ground truth in the batch: only the objectness term over the whole maps remains (loss.py:346-348)"""
    dev = p[0].device
    h = model.hyp
    gamma = _focal_gamma(model)
    obj_pw = torch.full((1,), float(h["obj_pw"]), device=dev)
    lobj = torch.zeros(1, device=dev)
    for pi in p:
        lobj = lobj + _obj_term(pi, torch.zeros_like(pi[..., 0]), obj_pw, gamma)
    lobj = lobj * h["obj"]
    zero = torch.zeros(1, device=dev)
    return lobj + zero, torch.cat((lobj, zero, zero, lobj)).detach()


def _obj_term(pi, tobj, obj_pw, gamma):
    """mean objectness BCE (focal when gamma is not None) over every cell of one head (model/loss.py:348)"""
    if gamma is None:
        return nn.functional.binary_cross_entropy_with_logits(pi[..., 5], tobj, pos_weight=obj_pw)
    e = nn.functional.binary_cross_entropy_with_logits(pi[..., 5], tobj, pos_weight=obj_pw, reduction="none")
    return _focal(e, gamma).mean()


def _sparse_terms(ps, r, model, h, cls_pw, gamma=None):
    """regression (+ class) loss of one head over ALL (anchor, target) rows weighted by the 0/1 assignment mask; ps =
    pi[b, a, gj, gi] with the unselected rows already zeroed.  Returns (lreg_i, lcls_i), unweighted.  gamma: the focal
    exponent of the SmoothL1 and class BCE terms (model/loss.py:286; the wh-IoU term is never focal), None = plain."""
    av, tbox = r["av"], r["tbox"]
    mf = r["mask"].to(ps.dtype)
    cnt = mf.sum().clamp(min=1.0)              # an empty selection contributes 0 like the reference's `if nb:`
    pxy = torch.sigmoid(ps[:, 0:2])
    pwh = torch.exp(ps[:, 2:4]).clamp(max=1e3) * av[:, :-1]
    pa = torch.atan(ps[:, 4]) + av[:, -1]
    liou = ((1.0 - wh_iou(tbox[:, 2:4], pwh)) * mf).sum() / cnt
    sm_xy = (_focal(nn.functional.smooth_l1_loss(pxy, tbox[:, 0:2], reduction="none"), gamma)
             * mf[:, None]).sum() / (2.0 * cnt)
    sm_a = (_focal(nn.functional.smooth_l1_loss(pa, tbox[:, 4], reduction="none"), gamma) * mf).sum() / cnt
    lreg = sm_xy + 2 * sm_a + liou * h["giou"]
    lcls = None
    if model.nc > 1:
        t = torch.zeros_like(ps[:, 6:])
        t[torch.arange(len(r["b"]), device=ps.device), r["tcls"]] = 1.0
        e = _focal(nn.functional.binary_cross_entropy_with_logits(ps[:, 6:], t, pos_weight=cls_pw, reduction="none"), gamma)
        lcls = (e * mf[:, None]).sum() / (cnt * e.shape[1])
    return lreg, lcls


def _tobj_of(pi, r):
    mf = r["mask"].to(pi.dtype)
    tobj = torch.zeros(pi.shape[:4], dtype=pi.dtype, device=pi.device)
    tobj.index_put_((r["b"], r["a"], r["gj"], r["gi"]), mf, accumulate=True)
    return tobj.clamp_(max=1.0)


def _compute_loss_masked(p, targets, model, hyp):
    dev = p[0].device
    h = model.hyp
    gamma = _focal_gamma(model)
    lcls = torch.zeros(1, device=dev)
    lobj = torch.zeros(1, device=dev)
    lreg = torch.zeros(1, device=dev)
    rows = _targets_masked(model, targets, hyp)
    # torch.full, not torch.tensor([...], device=...): the latter is a (synchronising) pageable host-to-device copy
    obj_pw = torch.full((1,), float(h["obj_pw"]), device=dev)
    cls_pw = torch.full((1,), float(h["cls_pw"]), device=dev)
    for pi, r in zip(p, rows):
        tobj = _tobj_of(pi, r)
        ps = pi[r["b"], r["a"], r["gj"], r["gi"]]
        # rows the reference never touches must not poison the sums: exp(inf) * 0 would be NaN in forward AND backward
        ps = torch.where(r["mask"][:, None], ps, torch.zeros_like(ps))
        lreg_i, lcls_i = _sparse_terms(ps, r, model, h, cls_pw, gamma)
        lreg = lreg + lreg_i
        if lcls_i is not None:
            lcls = lcls + lcls_i
        lobj = lobj + _obj_term(pi, tobj, obj_pw, gamma)
    lobj = lobj * h["obj"]
    lcls = lcls * h["cls"]
    lreg = lreg * h["reg"]
    loss = lobj + lcls + lreg
    return loss, torch.cat((lobj, lcls, lreg, loss)).detach()


def _targets_masked_stacked(model, targets, hyp):
    """_targets_masked with the per-layer loop folded into a leading layer dimension (the CUDA path: a third of the tiny
    element-wise launches).  Same element arithmetic; requires the same number of anchors in every YOLO layer.  Returns a
    dict of [nl, R] (R = na * nt, row = a * nt + t) tensors: b, a, gj, gi (int64), mask (bool), tbox [nl, R, 5],
    av [nl, R, 3], tcls [R]."""
    nt = len(targets)
    dev = targets.device
    layers = [model.module_list[i] for i in model.yolo_layers]
    nl = len(layers)
    av_all = torch.stack([l.anchor_vec.to(dev) for l in layers], 0)              # [nl, na, 3]
    ng = torch.stack([l.ng.to(dev) for l in layers], 0)                          # [nl, 2]
    na = av_all.shape[1]
    wh = []
    for _ in range(nl):        # the reference compounds the context factor once per layer (loss.py:186-187): keep the order
        targets[:, 4] += targets[:, 5] * (hyp["context_factor"] - 1)
        targets[:, 5] *= hyp["context_factor"]
        wh.append(targets[:, 4:6].clone())
    wh = torch.stack(wh, 0) * ng[:, None, :]                                     # [nl, nt, 2] in grid units
    ang = targets[:, 6]
    w1, h1 = av_all[:, :, 0:1], av_all[:, :, 1:2]                                # [nl, na, 1]
    w2, h2 = wh[:, None, :, 0], wh[:, None, :, 1]                                # [nl, 1, nt]
    inter = torch.min(w1, w2) * torch.min(h1, h2)
    all_ious = inter / ((w1 * h1 + 1e-16) + w2 * h2 - inter)                     # [nl, na, nt]
    gxy = targets[None, :, 2:4] * ng[:, None, :]                                 # [nl, nt, 2]
    gij = gxy.long()
    gfrac = gxy - gxy.floor()
    R = na * nt
    rep = lambda x: x[:, None].expand(nl, na, *x.shape[1:]).reshape(nl, R, *x.shape[2:])     # [nl, nt, ..] -> [nl, R, ..]
    a_idx = torch.arange(na, device=dev).view(-1, 1).expand(na, nt).reshape(-1)               # [R]
    gwha = torch.cat((wh, ang.view(1, nt, 1).expand(nl, nt, 1)), 2)              # [nl, nt, 3]
    tbox = torch.cat((rep(gfrac), rep(gwha)), 2)                                 # [nl, R, 5]
    av = av_all[:, a_idx]                                                        # [nl, R, 3]
    bc = targets[:, :2].long()
    b_idx = bc[:, 0].repeat(na)
    tcls = bc[:, 1].repeat(na)
    # angle gate with the LAST layer's anchor angles (the reference's loop variable after the loop, loss.py:222-224)
    angle_offset = (ang.view(1, nt) - av_all[-1, :, 2].view(na, 1)).abs()       # [na, nt]
    angle_offset = torch.where(angle_offset > 0.5 * math.pi, math.pi - angle_offset, angle_offset)
    j = (all_ious > model.hyp["iou_t"]) & (angle_offset < model.hyp["ang_t"])[None]          # [nl, na, nt]
    gt_any = j.any(1).any(0)                                                     # [nt]
    G = all_ious.reshape(nl * na, nt)
    cand = G == G.max(0)[0]
    layer_id = cand.float().argmax(0) // na
    angr = angle_offset.repeat(nl, 1)
    best = torch.where(cand, angr, torch.full_like(angr, float("inf"))).argmin(0)
    anchor = best % na
    onehot = torch.arange(na, device=dev).view(-1, 1) == anchor.view(1, -1)      # [na, nt]
    rescue = (~gt_any) & (torch.arange(nl, device=dev).view(-1, 1) == layer_id.view(1, -1))   # [nl, nt]
    mask = (j | (onehot[None] & rescue[:, None, :])).reshape(nl, R)
    ex = lambda x: x[None].expand(nl, R).contiguous()
    return dict(b=ex(b_idx), a=ex(a_idx), gj=rep(gij[..., 1:2]).reshape(nl, R).contiguous(),
                gi=rep(gij[..., 0:1]).reshape(nl, R).contiguous(), mask=mask, tbox=tbox, av=av, tcls=tcls, nl=nl, R=R)


def _sparse_terms_stacked(ps, r, model, h, cls_pw, gamma=None):
    """_sparse_terms over all layers at once: ps [nl, R, no]; returns (lreg, lcls) summed over the layers, unweighted"""
    av, tbox = r["av"], r["tbox"]
    mf = r["mask"].to(ps.dtype)                                                   # [nl, R]
    cnt = mf.sum(1).clamp(min=1.0)                                                # [nl]
    pxy = torch.sigmoid(ps[..., 0:2])
    pwh = torch.exp(ps[..., 2:4]).clamp(max=1e3) * av[..., :-1]
    pa = torch.atan(ps[..., 4]) + av[..., -1]
    w1, h1, w2, h2 = tbox[..., 2], tbox[..., 3], pwh[..., 0], pwh[..., 1]
    inter = torch.min(w1, w2) * torch.min(h1, h2)
    iou = inter / ((w1 * h1 + 1e-16) + w2 * h2 - inter)
    liou = ((1.0 - iou) * mf).sum(1) / cnt
    sm_xy = (_focal(nn.functional.smooth_l1_loss(pxy, tbox[..., 0:2], reduction="none"), gamma)
             * mf[..., None]).sum((1, 2)) / (2.0 * cnt)
    sm_a = (_focal(nn.functional.smooth_l1_loss(pa, tbox[..., 4], reduction="none"), gamma) * mf).sum(1) / cnt
    lreg = (sm_xy + 2 * sm_a + liou * h["giou"]).sum()
    lcls = None
    if model.nc > 1:
        nc = ps.shape[-1] - 6
        t = (torch.arange(nc, device=ps.device).view(1, 1, nc) == r["tcls"].view(1, -1, 1)).to(ps.dtype).expand(ps.shape[0], -1, -1)
        e = _focal(nn.functional.binary_cross_entropy_with_logits(ps[..., 6:], t, pos_weight=cls_pw, reduction="none"), gamma)
        lcls = ((e * mf[..., None]).sum((1, 2)) / (cnt * nc)).sum()
    return lreg, lcls


# ---------------------------------------------------------------------------------------------------------------
# CUDA path: the dense objectness term and the whole head cotangent in two hand-written kernels (csrc/loss.cu)
# ---------------------------------------------------------------------------------------------------------------
class _FusedLoss(torch.autograd.Function):
    """loss = obj * sum_i mean BCE(pi[..., 5], tobj_i) + reg * lreg + cls * lcls with the values of _compute_loss_masked.

    forward : the matched rows are gathered (tiny [na*nt, no] tensors) and their terms -- and the gradient with respect to
              the gathered rows -- evaluated with the same framework expressions as the masked form; the objectness term
              over all 35 M cells is ONE kernel per head reading the head tensor through its strides (so the permuted
              view of the NCHW buffer the head convolution wrote is consumed in place).
    backward: ONE kernel per head writes the whole cotangent (objectness channel, zeros elsewhere) with the strides of
              the input, the row gradients are scattered on top.  Nothing reads a device value on the host.
    gamma (focal arcs): the objectness kernels are the ryolo_obj_focal_* instantiations, the matched-row terms take
    the focal factor through _sparse_terms_stacked; None runs exactly the plain BCE path."""

    @staticmethod
    def _row_ptrs(r, m8, i):
        from . import _lib
        step = r["R"] * 8
        return (ctypes.c_void_p(r["b"].data_ptr() + i * step), ctypes.c_void_p(r["a"].data_ptr() + i * step),
                ctypes.c_void_p(r["gj"].data_ptr() + i * step), ctypes.c_void_p(r["gi"].data_ptr() + i * step),
                ctypes.c_void_p(m8.data_ptr() + i * r["R"]), int(r["R"]))

    @staticmethod
    def forward(ctx, model, r, h, gamma, *p):
        from . import _lib
        lib = _lib.lib
        dev = p[0].device
        st = _lib.stream_ptr(dev)
        no = p[0].shape[-1]
        lreg = torch.zeros(1, device=dev)
        lcls = torch.zeros(1, device=dev)
        tobjs, counts = [], []
        row_grads = m8 = None
        sums = torch.zeros(len(p), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            if r is not None:
                m8 = r["mask"].to(torch.uint8).contiguous()
                ps_all = torch.empty((r["nl"], r["R"], no), dtype=p[0].dtype, device=dev)
            for i, pi in enumerate(p):
                B, na, ny, nx, _ = pi.shape
                strides = (ctypes.c_longlong * 5)(*pi.stride())
                tobj = torch.zeros((B, na, ny, nx), dtype=pi.dtype, device=dev)
                if r is not None:
                    ra = _FusedLoss._row_ptrs(r, m8, i)
                    _lib.check(lib.ryolo_loss_rows_gather(_lib.ptr(pi), strides, B, na, ny, nx, no, *ra,
                                                          ctypes.c_void_p(ps_all[i].data_ptr()), st), "loss_rows_gather")
                    _lib.check(lib.ryolo_loss_rows_set_tobj(_lib.ptr(tobj), B, na, ny, nx, *ra, st), "loss_rows_set_tobj")
                if gamma is None:
                    _lib.check(lib.ryolo_obj_bce_fwd(_lib.ptr(pi), strides, B, na, ny, nx, no, 5, _lib.ptr(tobj),
                                                     float(h["obj_pw"]), ctypes.c_void_p(sums[i:].data_ptr()), st),
                               "obj_bce_fwd")
                else:
                    _lib.check(lib.ryolo_obj_focal_fwd(_lib.ptr(pi), strides, B, na, ny, nx, no, 5, _lib.ptr(tobj),
                                                       float(h["obj_pw"]), gamma, ctypes.c_void_p(sums[i:].data_ptr()),
                                                       st), "obj_focal_fwd")
                tobjs.append(tobj)
                counts.append(float(B * na * ny * nx))
            if r is not None:
                cls_pw = torch.full((1,), float(h["cls_pw"]), device=dev)
                with torch.enable_grad():
                    ps_all.requires_grad_()
                    lreg_s, lcls_s = _sparse_terms_stacked(ps_all, r, model, h, cls_pw, gamma)
                    sparse = lreg_s * h["reg"]
                    lreg = lreg + lreg_s.detach()
                    if lcls_s is not None:
                        sparse = sparse + lcls_s * h["cls"]
                        lcls = lcls + lcls_s.detach()
                    row_grads = torch.autograd.grad(sparse, ps_all)[0].contiguous()
        lobj = sums[0] * (h["obj"] / counts[0])          # python scalars only: no host-to-device copy, no sync
        for i in range(1, len(p)):
            lobj = lobj + sums[i] * (h["obj"] / counts[i])
        lobj = lobj.float().view(1)
        lreg = lreg * h["reg"]
        lcls = lcls * h["cls"]
        loss = lobj + lcls + lreg
        ctx.rows, ctx.tobjs, ctx.row_grads, ctx.counts, ctx.keep = r, tobjs, row_grads, counts, m8
        ctx.obj_w, ctx.obj_pw, ctx.gamma = float(h["obj"]), float(h["obj_pw"]), gamma
        ctx.save_for_backward(*p)
        items = torch.cat((lobj, lcls, lreg, loss)).detach()
        ctx.mark_non_differentiable(items)
        return loss, items

    @staticmethod
    def backward(ctx, gloss, _gitems):
        from . import _lib
        lib = _lib.lib
        p = ctx.saved_tensors
        dev = p[0].device
        gloss = gloss.reshape(-1)[:1].float().contiguous()
        st = _lib.stream_ptr(dev)
        grads = []
        with torch.cuda.device(dev):
            for i, pi in enumerate(p):
                B, na, ny, nx, no = pi.shape
                # the cotangent gets the memory layout of the input: for the permuted view of an NCHW head buffer (what
                # Darknet.forward returns) it reaches the network's backward as a contiguous NCHW tensor, no copy
                g = torch.empty_strided(pi.shape, pi.stride(), dtype=pi.dtype, device=dev)   # every element is written
                scale = gloss * (ctx.obj_w / ctx.counts[i])
                strides = (ctypes.c_longlong * 5)(*pi.stride())
                if ctx.gamma is None:
                    _lib.check(lib.ryolo_obj_bce_bwd(_lib.ptr(pi), strides, B, na, ny, nx, no, 5, _lib.ptr(ctx.tobjs[i]),
                                                     ctx.obj_pw, _lib.ptr(scale), _lib.ptr(g), st), "obj_bce_bwd")
                else:
                    _lib.check(lib.ryolo_obj_focal_bwd(_lib.ptr(pi), strides, B, na, ny, nx, no, 5, _lib.ptr(ctx.tobjs[i]),
                                                       ctx.obj_pw, ctx.gamma, _lib.ptr(scale), _lib.ptr(g), st),
                               "obj_focal_bwd")
                if ctx.rows is not None:
                    ra = _FusedLoss._row_ptrs(ctx.rows, ctx.keep, i)
                    _lib.check(lib.ryolo_loss_rows_scatter_add(_lib.ptr(g), strides, B, na, ny, nx, no, *ra,
                                                               ctypes.c_void_p(ctx.row_grads[i].data_ptr()), _lib.ptr(gloss),
                                                               st), "loss_rows_scatter_add")
                grads.append(g)
        return (None, None, None, None) + tuple(grads)


def _compute_loss_fused(p, targets, model, hyp):
    h = model.hyp
    gamma = _focal_gamma(model)
    nas = {int(pi.shape[1]) for pi in p}
    if len(nas) != 1 or len({int(pi.shape[-1]) for pi in p}) != 1:      # ragged anchor counts: the per-layer framework form
        return _compute_loss_masked(p, targets, model, hyp) if len(targets) else _compute_loss_no_targets(p, model)
    rows = _targets_masked_stacked(model, targets, hyp) if len(targets) else None
    return _FusedLoss.apply(model, rows, h, gamma, *p)
