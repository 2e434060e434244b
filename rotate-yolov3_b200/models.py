"""``Darknet(cfg, hyp, arc).forward`` behind the reference's signature (model/models.py:230-313), executed by
libryolo.so: every Conv2d -> BatchNorm2d -> PReLU block is one wgmma implicit-GEMM launch with BN folded, the
shortcut add / nearest-x2 upsample / channel concat of the graph fused into the producing conv's epilogue (residual
read, 2x2 replicated store, store at a channel offset of the shared concat buffer), and the YOLO heads decoded by one
fused kernel each.

What is kept from the reference so that train.py / test.py / detect.py see the same object:
  * ``module_defs`` / ``module_list`` / ``routes`` / ``yolo_layers`` / ``hyp`` / ``version`` / ``seen``;
  * parameter names: ``module_list.{i}.Conv2d.weight``, ``.BatchNorm2d.{weight,bias,running_mean,running_var,
    num_batches_tracked}``, ``.activation.weight`` (checkpoints and the optimizer split key on them, SURVEY.md 3.4);
  * YOLO layers expose ``ng, anchor_vec, anchor_wh, stride, nx, ny, na, nc`` (read by model/loss.py:172-174,313);
  * eval forward returns ``(io [B, sum(na*ny*nx), nc+6], (p0, p1, p2))`` with p_i = [B, na, ny, nx, nc+6].

Eval mode: inference path above.  Training mode: ``forward`` returns the list of raw head tensors like the reference
(models.py:192-194) and is differentiable -- forward with batch-statistics BatchNorm and the whole backward run on the
same library (train_path.py).  There is no PyTorch fallback in either mode."""
import ctypes

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from . import graph as G
from . import layout as L
from .parse_config import parse_model_cfg
from .pool import ActivationPool


class SELayer(nn.Module):
    """reference model/models.py:16-31 (same parameter names: fc.0.weight [c/r, c], fc.2.weight [c, c/r]); executed by
    ryolo_se_block / ryolo_se_fwd inside the eval plan and ryolo_se_fwd / ryolo_se_bwd inside the training plan, this
    forward exists only for module-tree parity."""

    def __init__(self, channel, reduction=16):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(nn.Linear(channel, channel // reduction, bias=False), nn.ReLU(inplace=True),
                                nn.Linear(channel // reduction, channel, bias=False), nn.Sigmoid())

    def forward(self, x):
        raise RuntimeError("SELayer runs inside Darknet's fused plan (libryolo.so), not as a stand-alone module")


class YOLOLayer(nn.Module):
    """reference model/models.py:170-227; decode runs in ryolo_yolo_decode."""

    def __init__(self, anchors, nc, yolo_index, arc, hyp):
        super().__init__()
        self.anchors = torch.Tensor(np.asarray(anchors, dtype=np.float64))
        self.na = len(anchors)
        self.nc = nc
        self.nx = 0
        self.ny = 0
        self.arc = arc
        self.hyp = hyp
        self.yolo_index = yolo_index

    def create_grids(self, img_size, ng, device, dtype=torch.float32):
        """reference model/model_utils.py:16-35 (without its in-place division bug on CPU: anchors are not
        modified, anchor_vec is a fresh tensor)."""
        nx, ny = ng
        self.img_size = max(img_size)
        self.stride = self.img_size / max(ng)
        yv, xv = torch.meshgrid([torch.arange(ny), torch.arange(nx)], indexing="ij")
        # non-blocking uploads: an eval loop that alternates sizes (detect.py --multi-scale) re-makes the grids at every
        # change of size and must not wait for the device each time
        self.grid_xy = torch.stack((xv, yv), 2).to(device, non_blocking=True).type(dtype).view((1, 1, ny, nx, 2))
        self.anchor_vec = self.anchors.clone().to(device, non_blocking=True)
        self.anchor_vec[:, :2] /= self.stride
        self.anchor_wh = self.anchor_vec.view(1, self.na, 1, 1, 3).to(device).type(dtype)
        self.ng = torch.Tensor(ng).to(device, non_blocking=True)
        self.nx = nx
        self.ny = ny
        a = self.anchors.to(device=device, dtype=torch.float32, non_blocking=True).contiguous()
        old = getattr(self, "_anchors_dev", None)
        if old is not None and old.device == a.device and old.shape == a.shape:
            # in place: the CUDA graphs of the eval plans of other shapes hold this address in their decode launches
            old.copy_(a)
        else:
            self._anchors_dev = a

    def decode_into(self, p, img_size, io, rows_total, row_offset):
        """p: [B, na*(nc+6), ny, nx] fp32 NCHW head output -> writes rows of io, returns the permuted raw view."""
        bs, ny, nx = p.shape[0], p.shape[-2], p.shape[-1]
        if (self.nx, self.ny) != (nx, ny) or getattr(self, "_anchors_dev", None) is None or \
                self._anchors_dev.device != p.device:
            self.create_grids(img_size, (nx, ny), p.device, p.dtype)
        # the raw head is handed out as the [B, na, ny, nx, no] VIEW of the NCHW buffer (model/models.py:190-192 without the
        # .contiguous() copy: a third of this kernel's traffic), like the training path
        st = _lib.lib.ryolo_yolo_decode(_lib.ptr(p), bs, self.na, self.nc, ny, nx, _lib.ptr(self._anchors_dev),
                                        float(self.stride), float(self.hyp["context_factor"]),
                                        1 if "default" in self.arc else 0, _lib.ptr(io), rows_total, row_offset,
                                        None, _lib.stream_ptr(p.device))
        _lib.check(st, "ryolo_yolo_decode")
        return p.view(bs, self.na, self.nc + 6, ny, nx).permute(0, 1, 3, 4, 2)

    def forward(self, p, img_size, var=None):
        if self.training:
            bs, ny, nx = p.shape[0], p.shape[-2], p.shape[-1]
            if (self.nx, self.ny) != (nx, ny):
                self.create_grids(img_size, (nx, ny), p.device, p.dtype)
            return p.view(bs, self.na, self.nc + 6, self.ny, self.nx).permute(0, 1, 3, 4, 2).contiguous()
        if "default" not in self.arc:
            raise NotImplementedError("only the 'default' arcs are decoded by the fused kernel")
        p = p.float().contiguous()
        bs, ny, nx = p.shape[0], p.shape[-2], p.shape[-1]
        rows = self.na * ny * nx
        io = torch.empty((bs, rows, self.nc + 6), dtype=torch.float32, device=p.device)
        pp = self.decode_into(p, img_size, io, rows, 0)
        return io, pp


def create_modules(module_defs, arc, hyp):
    """reference model/models.py:36-164 -- same module structure and names; smart bias init omitted (it always
    fails in the reference, models.py:132-155)."""
    hyperparams = module_defs.pop(0)
    output_filters = [int(hyperparams["channels"])]
    module_list = nn.ModuleList()
    routes = []
    yolo_index = -1
    filters = output_filters[-1]
    for i, mdef in enumerate(module_defs):
        modules = nn.Sequential()
        t = mdef["type"]
        if t == "convolutional":
            bn = int(mdef["batch_normalize"])
            filters = int(mdef["filters"])
            k = int(mdef["size"])
            pad = (k - 1) // 2 if int(mdef["pad"]) else 0
            modules.add_module("Conv2d", nn.Conv2d(output_filters[-1], filters, k, int(mdef["stride"]), pad, bias=not bn))
            if bn:
                modules.add_module("BatchNorm2d", nn.BatchNorm2d(filters, momentum=0.1))
            if mdef["activation"] == "leaky":
                modules.add_module("activation", nn.PReLU(num_parameters=1, init=0.10))
        elif t == "d-convolutional":
            # reference models.py:68-77: the block's own layers are an empty Conv2d, BatchNorm2d and LeakyReLU; the
            # forward runs only the conv with the weight of block `weight_from` (models.py:255-265)
            if "weight_from" not in mdef:
                raise NotImplementedError("[d-convolutional] block %d without weight_from (identity -> BN -> leaky) has "
                                          "no kernel" % i)
            if int(mdef["pad"]) != 1 or int(mdef["stride"]) != 1:
                raise NotImplementedError("[d-convolutional] block %d: only pad=1, stride=1 ('same' size) runs" % i)
            bn = int(mdef["batch_normalize"])
            filters = int(mdef["filters"])
            modules.add_module("Conv2d", nn.Sequential())
            if bn:
                modules.add_module("BatchNorm2d", nn.BatchNorm2d(filters, momentum=0.1))
            if mdef["activation"] == "leaky":
                modules.add_module("activation", nn.LeakyReLU(0.1, inplace=True))
        elif t == "maxpool":
            k, s = int(mdef["size"]), int(mdef["stride"])
            mp = nn.MaxPool2d(kernel_size=k, stride=s, padding=int((k - 1) // 2))
            if k == 2 and s == 1:
                modules.add_module("ZeroPad2d", nn.ZeroPad2d((0, 1, 0, 1)))
                modules.add_module("MaxPool2d", mp)
            else:
                modules = mp
        elif t == "upsample":
            modules = nn.Upsample(scale_factor=int(mdef["stride"]), mode="nearest")
        elif t == "se":
            modules = SELayer(int(mdef["channels"]))           # reference models.py:88-90
        elif t == "route":
            layers = [int(x) for x in mdef["layers"].split(",")]
            filters = sum(output_filters[l + 1 if l > 0 else l] for l in layers)
            routes.extend([l if l > 0 else l + i for l in layers])
        elif t == "shortcut":
            filters = output_filters[int(mdef["from"])]
            layer = int(mdef["from"])
            routes.extend([i + layer if layer < 0 else layer])
        elif t == "yolo":
            yolo_index += 1
            lo, hi = [int(v) for v in mdef["mask"].split("-")]
            modules = YOLOLayer(anchors=mdef["anchors"][lo:hi + 1], nc=int(mdef["classes"]), hyp=hyp,
                                yolo_index=yolo_index, arc=arc)
        else:
            raise NotImplementedError("layer type %r is outside the hot-path scope (SURVEY.md section 2)" % t)
        if "weight_from" in mdef:
            _check_shared_weight(module_defs, module_list, i, output_filters[-1], filters)
        module_list.append(modules)
        output_filters.append(filters)
    return module_list, routes


def _check_shared_weight(module_defs, module_list, i, cin, cout):
    """A `weight_from = j` block runs F.conv2d(x, module_list[j].Conv2d.weight) with stride 1 and no bias, BN or
    activation (reference models.py:255-265).  Only an earlier [convolutional] block that owns its weight may be j."""
    mdef, j = module_defs[i], int(module_defs[i]["weight_from"])
    if not (0 <= j < i and module_defs[j]["type"] == "convolutional" and "weight_from" not in module_defs[j]):
        raise NotImplementedError("block %d: weight_from=%d is not an earlier [convolutional] block with its own "
                                  "Conv2d" % (i, j))
    k = int(mdef["size"])
    if int(mdef["stride"]) != 1 or (k == 3 and int(mdef["pad"]) != 1):
        raise NotImplementedError("block %d: weight_from blocks run with stride 1 and 'same' padding only" % i)
    if tuple(module_list[j].Conv2d.weight.shape) != (cout, cin, k, k):
        raise ValueError("block %d: weight_from=%d has weight %s, the block needs %s" % (
            i, j, tuple(module_list[j].Conv2d.weight.shape), (cout, cin, k, k)))


class Darknet(nn.Module):
    def __init__(self, cfg, hyp, arc="default", precision="bf16"):
        """precision: "bf16" = throughput mode (bf16 operands / activations, fp32 accumulate); "parity" = fp32-grade
        arithmetic on the same tensor pipe (split bf16 operands, parity_path.py) for the reference's 1e-4 tolerance."""
        super().__init__()
        if precision not in ("bf16", "parity"):
            raise ValueError("precision must be 'bf16' or 'parity'")
        self.precision = precision
        self._pplan = None
        self._pplan_key = None
        self.module_defs = parse_model_cfg(cfg)
        self.net_hyper = self.module_defs[0]
        self.module_list, self.routes = create_modules(self.module_defs, arc, hyp)
        self.yolo_layers = [i for i, d in enumerate(self.module_defs) if d["type"] == "yolo"]
        self.hyp = hyp
        self.arc = arc
        self.version = np.array([0, 2, 5], dtype=np.int32)
        self.seen = np.array([0], dtype=np.int64)
        # Plans are cached per shape, (batch, h, w, device), and per mode; the shape-sized storage of all training plans
        # is one ActivationPool (pool.py), that of the eval plans one per batch size, so the plans of the reference's
        # multi-scale loops stay resident at the cost of the largest shape.  Eval plans hold weights packed at one parameter version (_plans_ver): a version change
        # drops them all.  _tshared / _eshared: the parameter-sized device state the plans of every shape share.
        self._plans, self._tplans, self._pools = {}, {}, {}
        self._plans_ver = None
        self._tshared, self._eshared = {}, {}
        self._plan_cur = self._tplan_cur = None
        self._ver_tensors = None
        # opt-in: replay the eval forward as ONE CUDA graph (78 launches -> 1).  The returned tensors are then static
        # buffers that the next forward overwrites (standard CUDA-graph semantics), hence not the default.
        self.use_cuda_graph = False
        self._graph = self._x_static = self._graph_out = self._graph_kernels = None
        self.replayed_kernels = 0

    # the plans of the last forward in each mode; assigning None drops the whole cache of that mode
    @property
    def _plan(self):
        return self._plan_cur

    @_plan.setter
    def _plan(self, value):
        if value is not None:
            raise ValueError("only None (drop the eval plans) can be assigned")
        self._drop_eval()
        self._eshared.clear()

    @property
    def _tplan(self):
        return self._tplan_cur

    @_tplan.setter
    def _tplan(self, value):           # `model._tplan = None`, the spelling bench.py uses
        if value is not None:
            raise ValueError("only None (drop the training plans) can be assigned")
        self.drop_training_plans()

    def drop_training_plans(self):
        """forget every training plan and the parameter-sized state they share (packed weights, gradient arenas,
        all-reduce buckets); the next training forward builds its plan afresh in the pool"""
        self._drop_train()
        self._tshared.clear()

    def _drop_eval(self, batch=None):
        """the eval plans (with their CUDA graphs) of one batch size, or all; the packed weights stay"""
        for key in [k for k in self._plans if batch is None or k[0] == batch]:
            del self._plans[key]
        if self._plan_cur is not None and not any(p is self._plan_cur for p in self._plans.values()):
            self._plan_cur = None
            self._graph = self._x_static = self._graph_out = self._graph_kernels = None

    def _drop_train(self):
        self._tplans.clear()
        self._tplan_cur = None

    def _pool(self, mode, device):
        if (mode, device) not in self._pools:
            self._pools[(mode, device)] = ActivationPool(device)
        return self._pools[(mode, device)]

    # ------------------------------------------------------------------------------------------------------
    def fuse(self):
        """reference models.py:300-313 folds BN into the convs module-by-module; here folding happens when the
        GEMM operands are packed (every eval forward uses folded weights), so this only drops the cache."""
        self._plan = None

    def train(self, mode=True):
        self._plan = None
        return super().train(mode)

    def load_state_dict(self, *a, **k):
        self._plan = None
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):      # .to() / .cuda() / .half() / .float(): storage changes without a version bump
        self._plan = None
        self._tplan = None
        self._pools = {}
        self._pplan = None
        self._ver_tensors = None
        return super()._apply(fn, *a, **k)

    def _packed(self, key, desc, wt, scale=None):
        """packed weight operand, shared by the eval plans of every shape until the parameters change"""
        k = key + (desc.cin, desc.cout, desc.ksize)
        if k not in self._eshared:
            self._eshared[k] = L.pack_weights(desc, wt, scale)
        return self._eshared[k]

    # ------------------------------------------------------------------------------------------------------
    def _folded(self, i, device):
        """(weight [cout,cin,k,k], per-filter scale or None, bias [cout], slope or None) with eval-mode BN folded
        per utils/torch_utils.py:45-69."""
        seq = self.module_list[i]
        conv = seq.Conv2d
        w = conv.weight.detach().float()
        if hasattr(seq, "BatchNorm2d"):
            bn = seq.BatchNorm2d
            scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
            bias = bn.bias.detach().float() - bn.running_mean.detach().float() * scale
            if conv.bias is not None:
                bias = bias + conv.bias.detach().float() * scale
        else:
            scale = None
            bias = conv.bias.detach().float() if conv.bias is not None else torch.zeros(w.shape[0], device=device)
        slope = float(seq.activation.weight.detach().float().item()) if hasattr(seq, "activation") else None
        return w, scale, bias, slope

    def _build_plan(self, batch, height, width, device, pool):
        """the eval forward at one shape: its shape-sized storage from `pool` (every zero-initialised buffer is rewritten
        by every forward before it is read or restored by the pool when the plan takes the storage over, as each
        allocation says), the packed weights from _packed"""
        g = G.Graph(self, height, width, ("se", "maxpool", "d-convolutional"), "block type %r has no sm_90a kernel yet")
        # producers write the real channels of the interior; halo and padding channels are restored
        bufs = G.Buffers(g, lambda h, w, cs: (pool.padded(batch, h, w, cs, None), None), 32)
        steps = []
        heads = []
        first_xs = None
        raw = {}          # owner block -> its RAW packed weight, shared by every `weight_from` use
        phase = {}        # (role, shape) -> phase-layout scratch of the dilated convs (the steps run in order)

        def phase_buf(role, nb, h, w, cs, c):
            key = (role, nb, h, w, cs)
            if key not in phase:
                phase[key] = pool.padded(nb, h, w, cs, c)     # split / conv write channels < c; the rest is restored
            return phase[key]

        for t, i in g.ops:
            if t in ("convolutional", "d-convolutional"):
                cv = g.convs[i]
                src = None if i == 0 else bufs.view(i - 1)
                cout, oh, ow, k, s = cv.cout, cv.oh, cv.ow, cv.k, cv.stride
                if cv.owner is not None:
                    # reference models.py:265: the owner's raw weight, no bias, BN or activation
                    wt = self.module_list[cv.owner].Conv2d.weight
                    scale, bias, slope = None, torch.zeros(cout, dtype=torch.float32, device=device), None
                else:
                    wt, scale, bias, slope = self._folded(i, device)
                if cv.dil is not None:
                    # dilated 3x3 = ordinary pad-1 3x3 conv on the dh*dw phase images (ryolo_dilate_split / _merge);
                    # the shortcut that follows it is added by the merge
                    dh, dw = cv.dil
                    nb, hp, wp = batch * dh * dw, -(-src.h // dh), -(-src.w // dw)
                    xp = phase_buf("x", nb, hp, wp, L.round_up(src.c, 64), src.c)
                    yp = phase_buf("y", nb, hp, wp, L.round_up(cout, 32), cout)
                    desc = L.make_desc(nb, hp, wp, src.c, xp.shape[-1], cout, yp.shape[-1], 3, 1, False, 0.0)
                    if cv.owner not in raw:
                        raw[cv.owner] = self._packed(("raw", cv.owner), desc, wt)
                    out = bufs.out(cv.mat)[0]
                    res = bufs.view(cv.shortcut) if cv.fuse_res else None
                    steps.append(("dsplit", dict(x=src.ptr, xcs=src.cs, h=src.h, w=src.w, c=src.c, dh=dh, dw=dw, xp=xp,
                                                 keep=src)))
                    steps.append(("conv", dict(desc=desc, x=xp.data_ptr(), w=raw[cv.owner], b=L.padded_bias(desc, bias),
                                               y=yp.data_ptr(), r=None, keep=(xp, yp))))
                    steps.append(("dmerge", dict(yp=yp, h=src.h, w=src.w, c=cout, dh=dh, dw=dw,
                                                 r=res.ptr if res is not None else None,
                                                 rcs=res.cs if res is not None else 0, y=out.ptr, ycs=out.cs,
                                                 keep=(res, out))))
                    continue
                if i == 0:
                    if not (k == 3 and s == 1 and wt.shape[1] == 3 and cout in (16, 32) and slope is not None):
                        raise NotImplementedError("first layer must be 3x3/1 conv, 3 -> 16|32 channels, leaky")
                    wf = (wt * scale.view(-1, 1, 1, 1)).contiguous() if scale is not None else wt.contiguous()
                    first_s2d = 1 in g.convs and g.convs[1].s2d and 0 not in self.routes
                    if first_s2d:
                        # layer 0 feeds only the stride-2 layer 1: write its output directly in that layer's
                        # space-to-depth layout (no [B, H+2, W+2, 32] tensor, no s2d pass over it)
                        first_xs = pool.padded(batch, height // 2, width // 2, L.round_up(4 * cout, 64), 4 * cout)
                        v = bufs.views[0] = G.View(None, 0, cout, height, width)
                    else:
                        v = bufs.out(0)[0]
                    steps.append(("first", dict(w=wf, b=bias.contiguous(), cout=cout, slope=slope, out=v, xs=first_xs)))
                    continue
                fuse_res, fuse_up, is_head = cv.fuse_res, cv.fuse_up, cv.is_head
                if src.c != wt.shape[1]:
                    raise RuntimeError("channel mismatch at block %d" % i)
                x_ptr = src.ptr
                if cv.s2d:
                    # 3x3/stride-2 as a 2x2-tap stride-1 conv on the space-to-depth copy of the input (1.78x instead of
                    # 4x MMA work; also removes the 32->64 channel padding of the first down-sampling layer)
                    if i == 1 and first_xs is not None:
                        xs = first_xs                      # already written by the first-layer kernel
                    else:
                        xs = pool.padded(batch, src.h // 2, src.w // 2, L.round_up(4 * src.c, 64), 4 * src.c)
                        steps.append(("s2d", dict(x=src.ptr, xcs=src.cs, h=src.h, w=src.w, c=src.c, xs=xs, keep=src)))
                    desc = L.make_desc(batch, src.h // 2, src.w // 2, 4 * src.c, xs.shape[-1], cout, 0, 2, 1,
                                       slope is not None, slope if slope is not None else 0.0, fuse_res, 0, fuse_up, is_head)
                    wt = L.s2d_weight(wt)
                    x_ptr = xs.data_ptr()
                else:
                    desc = L.make_desc(batch, src.h, src.w, src.c, src.cs, cout, 0, k, s, slope is not None,
                                       slope if slope is not None else 0.0, fuse_res, 0, fuse_up, is_head)
                res = None
                if is_head:
                    out = pool.take((batch, cout, oh, ow), torch.float32)      # every element written by the head conv
                    out_ptr = out.data_ptr()
                    heads.append((i, out))
                else:
                    out = bufs.out(cv.mat)[0]
                    desc.cout_stride = out.cs
                    out_ptr = out.ptr
                    if fuse_res:
                        res = bufs.view(cv.shortcut)
                        desc.res_stride = res.cs
                if cv.owner is not None:
                    if cv.owner not in raw:
                        raw[cv.owner] = self._packed(("raw", cv.owner), desc, wt)
                    pw = raw[cv.owner]
                else:
                    pw = self._packed(("folded", i), desc, wt, scale)
                pb = L.padded_bias(desc, bias)
                steps.append(("conv", dict(desc=desc, x=x_ptr, w=pw, b=pb, y=out_ptr,
                                           r=res.ptr if res is not None else None, keep=(src, res, out))))
            elif t == "se":
                src = bufs.view(i - 1)
                if src is None or src.c != int(g.defs[i]["channels"]):
                    raise NotImplementedError("[se] block at %d: no materialised input / channel mismatch" % i)
                fc = self.module_list[i].fc
                cr = fc[0].weight.shape[0]
                if (i - 1) in self.routes:
                    # the unscaled input is read again (the reference's *_se.cfg: the shortcut three blocks later adds it,
                    # concat routes read it): u = x * s goes to a buffer of its own
                    v = bufs.out(i)[0]
                    steps.append(("se_fwd", dict(x=src.ptr, xcs=src.cs, u=v.ptr, ucs=v.cs, h=src.h, w=src.w, c=src.c,
                                                 w1=fc[0].weight.detach().float().contiguous(),
                                                 w2=fc[2].weight.detach().float().contiguous(), cr=cr,
                                                 # outputs of ryolo_se_fwd and its workspace: written every forward
                                                 m=pool.take((batch * src.c,), torch.float32),
                                                 p=pool.take((batch * cr,), torch.float32),
                                                 s=pool.take((batch * src.c,), torch.float32),
                                                 ws=pool.take((_lib.lib.ryolo_se_workspace_bytes(batch, src.h, src.w,
                                                                                                 src.c, cr),), torch.uint8),
                                                 keep=(src, v))))
                    continue
                # otherwise the scale is applied IN PLACE: nothing else reads the unscaled tensor
                steps.append(("se", dict(x=src.ptr, xcs=src.cs, h=src.h, w=src.w, c=src.c,
                                         w1=fc[0].weight.detach().float().contiguous(),
                                         w2=fc[2].weight.detach().float().contiguous(), cr=fc[0].weight.shape[0],
                                         # ryolo_se_block zeroes sums and writes scale every forward
                                         sums=pool.take((batch * src.c,), torch.float32),
                                         scale=pool.take((batch * src.c,), torch.float32), keep=src)))
                bufs.views[i] = src
            else:                                        # maxpool
                src = bufs.view(i - 1)
                v = bufs.out(i)[0]
                steps.append(("maxpool", dict(x=src.ptr, xcs=src.cs, h=src.h, w=src.w, c=src.c,
                                              stride=int(g.defs[i]["stride"]), y=v.ptr, ycs=v.cs, keep=(src, v))))
        pool.channels(bufs.channels)
        rows = [self.module_list[j].na * g.shape[j][1] * g.shape[j][2] for j in self.yolo_layers]
        return dict(steps=steps, heads=heads, rows=rows, img=(height, width), graph=None)

    # ------------------------------------------------------------------------------------------------------
    def forward(self, x, var=None):
        if not x.is_cuda:
            raise RuntimeError("Darknet.forward needs a CUDA tensor (sm_90a kernels, no CPU fallback)")
        x = x.float().contiguous()
        b, _, h, w = x.shape
        key = (b, h, w, x.device)
        if self.precision == "parity":
            from .parity_path import DarknetParityFn, ParityPlan
            with torch.cuda.device(x.device):
                pkey = key + (self.training,)
                if self._pplan is None or self._pplan_key != pkey:
                    # drop the old plan first: at batch 16 x 608^2 the training plan and the next one (eval, or another
                    # multi-scale size) do not fit one 80 GB card together
                    self._pplan = self._pplan_key = None
                    self._pplan = ParityPlan(self, b, h, w, x.device, self.training)
                    self._pplan_key = pkey
                if self.training:
                    names = [n for n, _ in self.named_parameters()]
                    return list(DarknetParityFn.apply(self._pplan, x, names, *list(self.parameters())))
                with torch.no_grad():
                    heads = self._pplan.forward(x)
                    if not self.yolo_layers:
                        return [hd.clone() for hd in heads]
                    return self._decode_heads(heads, b, h, w, x.device)
        if self.training:
            # reference models.py:192-194, 290-292: list of raw [B, na, ny, nx, nc+6] tensors; differentiable
            from .train_path import DarknetTrainFn, TrainPlan
            with torch.cuda.device(x.device):
                plan = self._tplans.get(key)
                if plan is None:
                    pool = self._pool("train", x.device)
                    plan, halo = pool.build(lambda: TrainPlan(self, b, h, w, x.device, pool, self._tshared),
                                            self._drop_train)
                    plan.halo = halo
                    self._tplans[key] = plan
                self._tplan_cur = plan
                raw = DarknetTrainFn.apply(plan, x, *list(self.parameters()))     # fp32 NCHW head buffers
                outs = []
                for t, yi in zip(raw, self.yolo_layers):
                    layer = self.module_list[yi]
                    # model/models.py:190-192 without the .contiguous(): same values, the loss reads the view in place
                    outs.append(t.view(b, layer.na, layer.nc + 6, t.shape[2], t.shape[3]).permute(0, 1, 3, 4, 2))
                return outs
        with torch.cuda.device(x.device):
            # the plan holds PACKED (BN-folded, bf16) copies of the weights: rebuild it when any parameter or buffer was
            # modified in place since (optimizer step, manual edits); train()/eval()/load_state_dict drop it explicitly
            if self._ver_tensors is None:      # walking the module tree costs ~1 ms; the tensor objects are stable
                self._ver_tensors = list(self.parameters()) + list(self.buffers())
            ver = sum(t._version for t in self._ver_tensors)
            if ver != self._plans_ver:
                self._plan = None
                self._plans_ver = ver
            # one eval pool per batch size: a caller may keep the heads of one batch while it runs single images
            # (detect.py --multi-scale: batch 1 at changing sizes, one pool)
            pool = self._pool(("eval", b), x.device)
            plan = self._plans.get(key)
            if plan is None:
                plan, halo = pool.build(lambda: self._build_plan(b, h, w, x.device, pool), lambda: self._drop_eval(b))
                plan["halo"] = halo
                self._plans[key] = plan
            self._plan_cur = plan
            pool.activate(plan["halo"], _lib.stream_ptr(x.device))
            if self.use_cuda_graph:
                if plan["graph"] is None:
                    # the CUDA-graph input, copied before every replay; outside the pool: only plans that capture need it
                    plan["x_static"] = x.clone()
                    xs = plan["x_static"]
                    self._run_eval(xs, b, h, w)          # warm-up (attribute calls, lazy inits) outside capture
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    c0 = _lib.lib.ryolo_launch_count()
                    with torch.cuda.graph(g):
                        plan["graph_out"] = self._run_eval(xs, b, h, w)
                    plan["graph"] = g
                    plan["graph_kernels"] = int(_lib.lib.ryolo_launch_count() - c0)
                xs = plan["x_static"]
                self._graph, self._x_static = plan["graph"], xs
                self._graph_out, self._graph_kernels = plan["graph_out"], plan["graph_kernels"]
                xs.copy_(x)
                self._graph.replay()
                self.replayed_kernels += self._graph_kernels     # this library's kernels executed by the replay
                return self._graph_out
            return self._run_eval(x, b, h, w)

    def _run_eval(self, x, b, h, w):
        plan = self._plan
        lib = _lib.lib
        stream = _lib.stream_ptr(x.device)
        for kind, a in plan["steps"]:
            if kind == "maxpool":
                st = lib.ryolo_maxpool2x2(ctypes.c_void_p(a["x"]), a["xcs"], b, a["h"], a["w"], a["c"], a["stride"],
                                          ctypes.c_void_p(a["y"]), a["ycs"], stream)
                _lib.check(st, "ryolo_maxpool2x2")
            elif kind == "se":
                st = lib.ryolo_se_block(ctypes.c_void_p(a["x"]), a["xcs"], b, a["h"], a["w"], a["c"], _lib.ptr(a["w1"]),
                                        _lib.ptr(a["w2"]), a["cr"], _lib.ptr(a["sums"]), _lib.ptr(a["scale"]), stream)
                _lib.check(st, "ryolo_se_block")
            elif kind == "se_fwd":
                st = lib.ryolo_se_fwd(ctypes.c_void_p(a["x"]), a["xcs"], ctypes.c_void_p(a["u"]), a["ucs"], b, a["h"], a["w"],
                                      a["c"], _lib.ptr(a["w1"]), _lib.ptr(a["w2"]), a["cr"], _lib.ptr(a["m"]),
                                      _lib.ptr(a["p"]), _lib.ptr(a["s"]), _lib.ptr(a["ws"]), a["ws"].numel(), stream)
                _lib.check(st, "ryolo_se_fwd")
            elif kind == "s2d":
                st = lib.ryolo_space_to_depth(ctypes.c_void_p(a["x"]), a["xcs"], b, a["h"], a["w"], a["c"],
                                              _lib.ptr(a["xs"]), a["xs"].shape[-1], stream)
                _lib.check(st, "ryolo_space_to_depth")
            elif kind == "dsplit":
                st = lib.ryolo_dilate_split(ctypes.c_void_p(a["x"]), a["xcs"], b, a["h"], a["w"], a["c"], a["dh"], a["dw"],
                                            _lib.ptr(a["xp"]), a["xp"].shape[-1], stream)
                _lib.check(st, "ryolo_dilate_split")
            elif kind == "dmerge":
                st = lib.ryolo_dilate_merge(_lib.ptr(a["yp"]), a["yp"].shape[-1], b, a["h"], a["w"], a["c"], a["dh"],
                                            a["dw"], ctypes.c_void_p(a["r"]) if a["r"] else None, a["rcs"], 0,
                                            ctypes.c_void_p(a["y"]), a["ycs"], stream)
                _lib.check(st, "ryolo_dilate_merge")
            elif kind == "first":
                if a["xs"] is not None:
                    st = lib.ryolo_conv_first_s2d_fwd(_lib.ptr(x), b, h, w, _lib.ptr(a["w"]), _lib.ptr(a["b"]),
                                                      a["cout"], a["slope"], _lib.ptr(a["xs"]), a["xs"].shape[-1], stream)
                else:
                    v = a["out"]
                    st = lib.ryolo_conv_first_fwd(_lib.ptr(x), b, h, w, _lib.ptr(a["w"]), _lib.ptr(a["b"]), a["cout"],
                                                  a["slope"], ctypes.c_void_p(v.ptr), v.cs, stream)
                _lib.check(st, "ryolo_conv_first_fwd")
            else:
                st = lib.ryolo_conv_bn_act_fwd(ctypes.byref(a["desc"]), ctypes.c_void_p(a["x"]), _lib.ptr(a["w"]),
                                               _lib.ptr(a["b"]), ctypes.c_void_p(a["r"]) if a["r"] else None,
                                               ctypes.c_void_p(a["y"]), stream)
                _lib.check(st, "ryolo_conv_bn_act_fwd")
        if not self.yolo_layers:      # trunk graph without YOLO layers: the raw head maps [B, filters, ny, nx]
            return [head for _, head in plan["heads"]]
        return self._decode_heads([head for _, head in plan["heads"]], b, h, w, x.device)

    def _decode_heads(self, heads, b, h, w, device):
        """fp32 NCHW head maps -> (io [B, sum(na*ny*nx), nc+6], (p0, p1, p2)) like models.py:294-298"""
        nc = self.module_list[self.yolo_layers[0]].nc
        rows = [self.module_list[yi].na * hd.shape[2] * hd.shape[3] for yi, hd in zip(self.yolo_layers, heads)]
        total = sum(rows)
        io = torch.empty((b, total, nc + 6), dtype=torch.float32, device=device)
        ps = []
        off = 0
        for head, yi, r in zip(heads, self.yolo_layers, rows):
            ps.append(self.module_list[yi].decode_into(head, (h, w), io, total, off))
            off += r
        return io, tuple(ps)
