"""TEST INFRASTRUCTURE: a float64 restatement of the training loss (the fused path of loss.compute_loss for the arcs
containing 'default'), the magnitudes of its fp32 terms and the checks of the loss value and the head cotangent against
it; targets that reach every branch of the loss; the reference's hyp.txt reader.  Shared by test_multiclass_f64_gpu.py
(which states the bounds) and test_se_f64_gpu.py (the same bounds at the reference's positive weights: every bound
carries lw = 1 + (pw - 1) t).  A single-class model (nc = 1) has no class term, as in the reference (`if model.nc > 1`):
its class column's cotangent is exactly 0."""
import torch

from f64_refs import F64, TINY, U

U64 = 2.0 ** -53
K_OBJ = 8          # fp32 roundings of one objectness term or its derivative (loss.cu), in units of U * magnitude
K_ROW = 16         # fp32 roundings of one matched-row term or its derivative (torch's fp32 autograd of the loss)


def _loss():
    from rotate_yolov3_b200 import loss
    return loss


def read_hyp(path):
    """a hyp.txt of the reference's recipes (utils/utils.py hyp_parse): `key: value  # comment` lines, each value a
    number or a Python expression"""
    hyp = {}
    with open(path) as f:
        for line in f:
            if line.startswith("#") or not line.strip():
                continue
            k, v = line.strip().split(":", 1)
            v = v.strip().split(" ")[0]
            try:
                hyp[k] = float(v)
            except ValueError:
                hyp[k] = float(eval(v))
    return hyp


def make_targets(model, nc, batch, h, w, seed):
    """[nt, 7] = (image, class, x, y, w, h, theta): the (w, h, theta) of a random anchor of any head, jittered by up to
    10 % and 3 degrees, so that every target has matched rows; five targets per image with classes 0, nc - 1 and values
    in between; image 0's last target is its first one in another class (two or more matched rows on each of its cells);
    the last image's last target sits on the right border (x = 1: its rows fall outside every map)"""
    g = torch.Generator().manual_seed(seed)
    anchors = torch.cat([model.module_list[i].anchors for i in model.yolo_layers]).float()
    rows = []
    for b in range(batch):
        for k in range(5):
            a = anchors[int(torch.randint(0, len(anchors), (1,), generator=g))]
            s = 1 + 0.1 * (2 * torch.rand(3, generator=g) - 1)
            xy = 0.05 + 0.9 * torch.rand(2, generator=g)
            cls = [0, nc - 1, (3 * b + 5 * k) % nc, (7 * b + k + 1) % nc, nc // 2][k]
            rows.append([b, cls, float(xy[0]), float(xy[1]), float(a[0] * s[0] / w), float(a[1] * s[1] / h),
                         float(a[2] + 0.05 * (s[2] - 1) * 10)])
    rows[4] = list(rows[0])
    rows[4][1] = (rows[0][1] + nc // 3) % nc
    rows[-1][2] = 1.0
    return torch.tensor(rows, dtype=torch.float32)


# ---------------------------------------------------------------------------------------------------------------
# float64 restatement of the loss and magnitudes of the fp32 path's terms
def _live(r, shape):
    """rows with mask = 1 whose cell lies inside the map (the fused path gathers 0 for a row outside and writes nothing
    for it; the reference raises an IndexError there), and the clamped indices"""
    B, na, ny, nx = shape[:4]
    inb = (r["gj"] >= 0) & (r["gj"] < ny) & (r["gi"] >= 0) & (r["gi"] < nx)
    return r["mask"] & inb, r["gj"].clamp(0, ny - 1), r["gi"].clamp(0, nx - 1)


def _bce_mag(x, t, pw):
    """magnitude of the terms of BCE with logits: |(1 - t) x| + lw (log1p(exp(-|x|)) + max(-x, 0))"""
    lw = 1 + (pw - 1) * t
    return ((1 - t) * x).abs() + lw * (torch.log1p(torch.exp(-x.abs())) + (-x).clamp_min(0))


def _sl1_mag(p, t):
    return (p.abs() + t.abs()) * (p.abs() + t.abs() + 1)


def loss64(p64, targets, model, hyp, shift_cls=0):
    """_compute_loss_masked in float64 (the same target assignment, _sparse_terms and _obj_term) on p64, with the fused
    path's convention for rows outside the map.  Returns (lobj, lcls, lreg) and the rows.  shift_cls: the one-hot
    shifted by that many columns (the bound self-test)."""
    L = _loss()
    h = model.hyp
    rows = L._targets_masked(model, targets.clone(), hyp)
    obj_pw = torch.full((1,), float(h["obj_pw"]), dtype=F64)
    cls_pw = torch.full((1,), float(h["cls_pw"]), dtype=F64)
    lobj = lcls = lreg = torch.zeros(1, dtype=F64)
    for pi, r in zip(p64, rows):
        live, gj, gi = _live(r, pi.shape)
        tobj = torch.zeros(pi.shape[:4], dtype=F64)
        tobj.index_put_((r["b"], r["a"], gj, gi), live.to(F64), accumulate=True)
        tobj = tobj.clamp(max=1.0)
        ps = torch.where(live[:, None], pi[r["b"], r["a"], gj, gi], torch.zeros((), dtype=F64))
        rr = dict(r, tcls=(r["tcls"] + shift_cls) % model.nc)
        lreg_i, lcls_i = L._sparse_terms(ps, rr, model, h, cls_pw)
        lreg = lreg + lreg_i
        if lcls_i is not None:                     # nc = 1: no class term
            lcls = lcls + lcls_i
        lobj = lobj + L._obj_term(pi, tobj, obj_pw, None)
    return (lobj * h["obj"], lcls * h["cls"], lreg * h["reg"]), rows


def magnitudes(p64, rows, model):
    """per head: M [B, na, ny, nx, no] (the objectness channel: scale (|1 - t| + lw (s + |s - 1|)); a matched cell's
    other channels: the sum over its rows of the magnitude of each row's derivative), the rows per cell, the live
    mask, and the magnitudes of the loss terms (lobj, lcls, lreg) for the value bounds"""
    h = model.hyp
    nc = model.nc
    out = []
    mag_loss = torch.zeros(3, dtype=F64)
    with torch.no_grad():
        for pi, r in zip(p64, rows):
            pi = pi.detach()
            B, na, ny, nx, no = pi.shape
            live, gj, gi = _live(r, pi.shape)
            tobj = torch.zeros(pi.shape[:4], dtype=F64)
            tobj.index_put_((r["b"], r["a"], gj, gi), live.to(F64), accumulate=True)
            tobj = tobj.clamp(max=1.0)
            count = B * na * ny * nx
            x = pi[..., 5]
            s = torch.sigmoid(x)
            lw = 1 + (h["obj_pw"] - 1) * tobj
            m = torch.zeros_like(pi)
            m[..., 5] = h["obj"] / count * ((1 - tobj).abs() + lw * (s + (s - 1).abs()))
            mag_loss[0] += h["obj"] / count * float(_bce_mag(x, tobj, h["obj_pw"]).sum())
            # matched rows (rows with mask = 1 count in cnt even outside the map, as in the fused path)
            ps = torch.where(live[:, None], pi[r["b"], r["a"], gj, gi], torch.zeros((), dtype=F64))
            mf = r["mask"].to(F64)
            cnt = float(mf.sum().clamp(min=1.0))
            av, tb = r["av"].double(), r["tbox"].double()
            c_reg = h["reg"] / cnt
            mr = torch.zeros((len(mf), no), dtype=F64)
            sg = torch.sigmoid(ps[:, 0:2])
            # the fp32 target offset is (t ng) - floor(t ng): it carries U (cell index + offset); torch's sigmoid
            # backward multiplies by (1 - s) s of the fp32 s, and 1 - s carries U s, not U (1 - s)
            txy = tb[:, 0:2].abs() + torch.stack((r["gi"], r["gj"]), 1).double().abs()
            mr[:, 0:2] = c_reg / 2 * (sg + txy) * sg
            ex = torch.exp(ps[:, 2:4])
            w2, h2 = ex[:, 0] * av[:, 0], ex[:, 1] * av[:, 1]
            w1, h1 = tb[:, 2], tb[:, 3]
            inter = torch.minimum(w1, w2) * torch.minimum(h1, h2)
            den = w1 * h1 + 1e-16 + w2 * h2 - inter
            a_, b_ = 1 / den + inter / den ** 2, inter / den ** 2
            cg = h["giou"] * c_reg
            mr[:, 2] = cg * w2 * (a_ * torch.minimum(h1, h2) * (w2 < w1) + b_ * h2) * (ex[:, 0] <= 1e3)
            mr[:, 3] = cg * h2 * (a_ * torch.minimum(w1, w2) * (h2 < h1) + b_ * w2) * (ex[:, 1] <= 1e3)
            at = torch.atan(ps[:, 4]).abs() + av[:, 2].abs()
            mr[:, 4] = 2 * c_reg * (at + tb[:, 4].abs()) / (1 + ps[:, 4] ** 2)
            if nc > 1:                             # nc = 1: no class term, the class column's cotangent is 0
                t1 = torch.zeros((len(mf), nc), dtype=F64)
                t1[torch.arange(len(mf)), r["tcls"]] = 1.0
                sc = torch.sigmoid(ps[:, 6:])
                mr[:, 6:] = h["cls"] / (cnt * nc) * (sc + h["cls_pw"] * t1)
            mr = mr * mf[:, None]
            # value magnitudes: class BCE terms; SmoothL1 (xy, theta) and 1 - iou
            if nc > 1:
                mag_loss[1] += h["cls"] / (cnt * nc) * float((_bce_mag(ps[:, 6:], t1, h["cls_pw"]) * mf[:, None]).sum())
            iou = inter / den
            reg_rows = (_sl1_mag(sg, txy).sum(1) / 2 + 2 * _sl1_mag(at, tb[:, 4]) + h["giou"] * (1 + iou)) * mf
            mag_loss[2] += c_reg * float(reg_rows.sum())
            # into the cells (live rows only), with the number of rows per cell
            mr[:, 5] = 0.0
            ncell = torch.zeros(pi.shape[:4], dtype=F64)
            idx = (r["b"][live], r["a"][live], gj[live], gi[live])
            ncell.index_put_(idx, torch.ones(int(live.sum()), dtype=F64), accumulate=True)
            mrow = torch.zeros_like(pi)
            mrow.index_put_(idx, mr[live], accumulate=True)
            m = m + mrow * (K_ROW + ncell[..., None]) / K_OBJ        # cot_check divides by K_OBJ U
            out.append(dict(m=m, ncell=ncell, live=live, n_rows=len(mf) * nc, cells=count))
    return out, mag_loss


def cot_check(got, want, mag, ncell):
    """the cotangent of one head [B, na, ny, nx, no]: worst |err| / (K_OBJ U M) over the objectness channel, the class
    columns and the regression columns of the matched cells; every other element exactly 0"""
    err = (got.double() - want).abs() / (K_OBJ * U * mag + TINY)
    matched = ncell > 0
    r = {"obj": float(err[..., 5].max()),
         "cls": float(err[..., 6:][matched].max()) if bool(matched.any()) else 0.0,
         "reg": float(err[..., :5][matched].max()) if bool(matched.any()) else 0.0}
    rest = torch.ones(got.shape, dtype=torch.bool)
    rest[..., 5] = False
    rest[matched] = False
    r["zero"] = bool((got[rest] == 0).all()) and bool((want[rest] == 0).all())
    r["matched_cells"] = int(matched.sum())
    return r


def loss_checks(st):
    """the loss value against float64 and the head cotangent, element by element"""
    lobj, lcls, lreg = (float(v) for v in st.want_items)
    got = st.items
    m0, m1, m2 = (float(v) for v in st.mag_loss)
    n_cls = max(mg["n_rows"] for mg in st.mags)
    n_reg = 2 * n_cls // st.nc
    # lobj: K_OBJ roundings per fp32 term, the double sums (a chain no longer than the cells), the float conversion;
    # lcls / lreg: K_ROW per term, a sequential fp32 sum over the rows (worst case), the divide, the layer adds, the weight
    cells = sum(mg["cells"] for mg in st.mags)
    b_obj = K_OBJ * U * m0 + cells * U64 * m0 + U * abs(lobj)
    b_cls = (K_ROW + n_cls + 8) * U * m1
    b_reg = (K_ROW + n_reg + 8) * U * m2
    # (+ TINY: nc = 1 has no class term, lcls and its bound are 0)
    st.loss_r = {"lobj": abs(float(got[0]) - lobj) / b_obj, "lcls": abs(float(got[1]) - lcls) / (b_cls + TINY),
                 "lreg": abs(float(got[2]) - lreg) / b_reg,
                 "loss": abs(float(got[3]) - (lobj + lcls + lreg)) / (b_obj + b_cls + b_reg
                                                                      + 2 * U * (abs(lobj) + abs(lcls) + abs(lreg)))}
    st.cot_r = {}
    for blk, g64, mg in zip(st.plan.heads, st.g64, st.mags):
        got_c = st.cot[blk.i]
        st.cot_r[blk.i] = cot_check(got_c, g64, mg["m"], mg["ncell"])
    hd = st.plan.heads[-1]
    st.stash["cot"] = dict(i=hd.i, got=st.cot[hd.i], want=st.g64[-1], m=st.mags[-1]["m"], ncell=st.mags[-1]["ncell"],
                           p32=st.p32)
    st.max_rows_per_cell = max(float(mg["ncell"].max()) for mg in st.mags)
    st.border_rows = sum(int((r["mask"] & ~mg["live"]).sum()) for r, mg in zip(st.rows, st.mags))


# ---------------------------------------------------------------------------------------------------------------
# the loss of a checked training step (checked_step.run_step's loss and head_grads hooks)
def fused_loss(st, ps, hyp):
    """the fused loss on the heads of this forward (st.targets); the float64 restatement on the same fp32 heads, its
    gradient, the magnitudes, and whether the fp32 assignment of the fused path equals the float64 one"""
    model, dev = st.model, ps[0].device
    st.p32 = [p.detach().cpu() for p in ps]
    loss, items = _loss().compute_loss(ps, st.targets.clone().to(dev), model, hyp)
    st.items = items.cpu().double()
    p64 = [p.double().requires_grad_(True) for p in st.p32]
    comps, rows = loss64(p64, st.targets.double(), model, hyp)
    sum(comps).sum().backward()
    st.want_items = torch.cat([c.detach() for c in comps])
    st.g64 = [p.grad for p in p64]
    st.rows = rows
    st.mags, st.mag_loss = magnitudes(p64, rows, model)
    fr = _loss()._targets_masked_stacked(model, st.targets.clone().to(dev), hyp)
    st.masks_equal = all(torch.equal(fr["mask"][l].cpu(), r["mask"]) for l, r in enumerate(rows))
    return loss


def record_head_grads(st, grads):
    """the head cotangents the plan receives: as the heads' dz layout (st.g_nhwc) and as [B, na, ny, nx, no] (st.cot)"""
    st.g_nhwc = {}
    for blk, g in zip(st.plan.heads, grads):
        g = g.contiguous()
        st.g_nhwc[blk.i] = g.permute(0, 2, 3, 1)
        st.cot[blk.i] = g.view(st.batch, -1, st.nc + 6, blk.oh, blk.ow).permute(0, 1, 3, 4, 2).cpu()
