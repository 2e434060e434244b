"""Parity-precision execution of ``Darknet`` (``Darknet(cfg, hyp, arc, precision="parity")``), eval and training mode.

The reference computes its Conv2d -> BatchNorm2d -> PReLU blocks in fp32 (model/models.py:55-65; apex O1 is optional,
train.py:165-166), and north_star asks for 1e-4 relative on conv activations.  This path meets that on the SAME tensor
pipe: GEMM operands are split into three bf16 planes (all 24 significant bits), a*w is evaluated as six exact-product
terms accumulated in fp32 with round-to-nearest segment sums (csrc/conv_parity.cu), everything between two GEMMs is
fp32 with fp64 reductions (csrc/parity.cu).  The bf16 path (models.py / train_path.py) stays the throughput mode; every
number bench.py prints says which precision produced it.

Per conv block, forward:  [space-to-depth of both planes] -> px_conv -> z (fp32) -> batch or running statistics ->
y = prelu(z*scale + shift) [+ shortcut] [2x2 replicated], re-split.  Backward: px_bn_act_bwd (fp32 dy, z -> d gamma,
d beta, d slope, split dz, shortcut gradient) -> wgrad (px_wgrad: the wgmma wgrad GEMM with segment sums, over all
planes of dz and x: nine plane blocks, summed by px_unpack_wgrad) -> dgrad (px_conv with mirrored / transposed split weights, fp32 accumulate
into the source's gradient buffer)."""
import ctypes
import weakref

import torch

from . import _lib
from . import graph as G
from . import layout as L
from .train_path import check_activations

NP = 3             # bf16 planes per operand: 3 = all 24 bits of an fp32 (2 = 16 bits: enough for eval, not for training BN)


def _terms(planes):
    """(a plane, w plane) pairs with i + j < planes, smallest magnitude first; returned as (count, a code, w code) with
    2 bits per term"""
    pairs = sorted(((i, j) for i in range(planes) for j in range(planes) if i + j < planes), key=lambda t: -(t[0] + t[1]))
    a = sum(i << (2 * t) for t, (i, _) in enumerate(pairs))
    w = sum(j << (2 * t) for t, (_, j) in enumerate(pairs))
    return len(pairs), a, w


NTERMS, A_CODE, W_CODE = _terms(NP)


def _lo(v):
    """channel stride of one plane of a split bf16 view: plane k of the activation starts at channel ch_off + k * _lo(v)"""
    return v.cs // NP


def _split_buf(batch, h, w, plane, device):
    return torch.zeros((batch, h + 2, w + 2, NP * plane), dtype=torch.bfloat16, device=device)


def _f32_buf(batch, h, w, cs, device):
    return torch.zeros((batch, h + 2, w + 2, cs), dtype=torch.float32, device=device)


class ParityPlan:
    def __init__(self, model, batch, height, width, device, train):
        self.model, self.batch, self.h, self.w, self.device, self.train = model, batch, height, width, device, train
        self.gen = 0            # forward generation (DarknetParityFn checks that backward sees the activations it saved)
        self.consumed = True
        if any(d["type"] == "se" for d in model.module_defs):
            raise NotImplementedError("[se] blocks have no parity-precision kernel; SE graphs run in precision='bf16'")
        g = G.Graph(model, height, width, (), "block type %r has no parity-precision kernel")
        if any(cv.stride == 2 and (cv.ih % 2 or cv.iw % 2) for cv in g.convs.values()):
            raise NotImplementedError("parity precision: stride-2 convs need even input sizes")
        # activations in split bf16 buffers [B, H+2, W+2, NP*P] (plane k at channel ch_off + k*P), gradients fp32
        bufs = G.Buffers(g, lambda hh, ww, plane: (_split_buf(batch, hh, ww, plane, device),
                                                   _f32_buf(batch, hh, ww, plane, device) if train else None), 64)

        self.col = _split_buf(batch, height, width, 64, device)     # im2col of the image: 27 real channels per plane
        blocks = []
        for _, i in g.ops:
            seq = model.module_list[i]
            b = g.convs[i]
            b.po = L.round_up(b.cout, 64)
            if i == 0:
                if not (b.k == 3 and b.stride == 1 and seq.Conv2d.weight.shape[1] == 3):
                    raise NotImplementedError("first layer must be a 3x3 stride-1 conv on 3 channels")
                b.src, b.gsrc = G.View(self.col, 0, 27, height, width), None
                b.k_eff = 1
            else:
                b.src, b.gsrc = bufs.view(i - 1), bufs.gview(i - 1)
                b.k_eff = b.k
            b.cin = b.src.c
            b.s2d = i > 0 and b.stride == 2 and b.k == 3
            if b.stride == 2 and not b.s2d:
                raise NotImplementedError("parity precision: only 3x3 stride-2 convs")
            if b.s2d:
                b.p4 = L.round_up(4 * b.cin, 64)
                b.xs = _split_buf(batch, b.src.h // 2, b.src.w // 2, b.p4, device)
                b.dxs = _f32_buf(batch, b.src.h // 2, b.src.w // 2, b.p4, device) if train else None
                b.k_eff = 2
                b.gh, b.gw_ = b.src.h // 2, b.src.w // 2          # GEMM grid
                b.cin_eff = 4 * b.cin
            else:
                b.gh, b.gw_ = b.src.h, b.src.w
                b.cin_eff = b.cin
            b.z = _f32_buf(batch, b.oh, b.ow, b.po, device)
            if b.is_head:
                b.out = torch.empty((batch, b.cout, b.oh, b.ow), dtype=torch.float32, device=device)
                b.res = b.gres = None
            else:
                if not b.has_bn:
                    raise NotImplementedError("conv block without BatchNorm that is not a YOLO head")
                b.y, b.gy = bufs.out(b.mat)
                if b.fuse_res:
                    b.res, b.gres = bufs.view(b.shortcut), bufs.gview(b.shortcut)
                else:
                    b.res = b.gres = None
                b.sums = torch.zeros(2 * b.cout, dtype=torch.float64, device=device)
                b.mean, b.invstd, b.scale, b.shift = (torch.zeros(b.cout, dtype=torch.float32, device=device)
                                                      for _ in range(4))
            b.pw = torch.empty(_lib.lib.ryolo_px_packed_weight_bytes(b.cout, b.cin_eff, b.k_eff, NTERMS),
                               dtype=torch.uint8, device=device)
            b.pw_ver = None
            if train:
                b.bsums = torch.zeros(2 * b.cout + 1, dtype=torch.float64, device=device)
                # wgrad over all planes of dz and of the WHOLE source buffer (a slice of a concat buffer is picked
                # out by px_unpack_wgrad's cin_off)
                b.xw_buf = b.xs if b.s2d else b.src.buf
                b.dz_shape = (batch, b.oh + 2, b.ow + 2, NP * b.po)
                b.dw_shape = (b.k_eff * b.k_eff, NP * b.po, b.xw_buf.shape[-1])
                if i > 0:
                    b.pwd = torch.empty(_lib.lib.ryolo_px_packed_weight_bytes(b.cin_eff, b.cout, b.k_eff, NTERMS),
                                        dtype=torch.uint8, device=device)
            blocks.append(b)
        self.blocks = blocks
        self.heads = [b for b in blocks if b.is_head]
        if train:
            # dz (split gradient of a block's raw conv output) and dw (plane blocks of the weight gradient) live only
            # inside their own block's backward: ONE scratch of the largest size each, re-viewed per block (a per-block
            # allocation costs 34 GB at batch 64).  Head blocks keep their own dz: all head gradients arrive before the
            # first block runs.
            import math
            dz_max = max(math.prod(b.dz_shape) for b in blocks if not b.is_head)
            dw_max = max(math.prod(b.dw_shape) for b in blocks)
            self._dz_scratch = torch.zeros(dz_max, dtype=torch.bfloat16, device=device)
            self._dw_scratch = torch.zeros(dw_max, dtype=torch.float32, device=device)
            for b in blocks:
                if b.is_head:
                    b.dz = torch.zeros(b.dz_shape, dtype=torch.bfloat16, device=device)
                    b.dz_shared = False
                else:
                    b.dz = self._dz_scratch[:math.prod(b.dz_shape)].view(b.dz_shape)
                    b.dz_shared = True
                b.dw = self._dw_scratch[:math.prod(b.dw_shape)].view(b.dw_shape)
            written = {}
            for b in reversed(blocks):
                b.gres_acc = G.claim(written, b.gres) if b.gres is not None else False
                b.gsrc_acc = G.claim(written, b.gsrc) if b.gsrc is not None else False

    # ------------------------------------------------------------------------------------------------------
    def forward(self, x):
        m, lib, B = self.model, _lib.lib, self.batch
        st = _lib.stream_ptr(self.device)
        vp = ctypes.c_void_p
        _lib.check(lib.ryolo_px_im2col_first(_lib.ptr(x), B, self.h, self.w, _lib.ptr(self.col), self.col.shape[-1], 64, NP, st),
                   "px_im2col_first")
        bn_counters = []
        for b in self.blocks:
            seq = m.module_list[b.i]
            w = seq.Conv2d.weight
            if w.dtype != torch.float32:
                raise NotImplementedError("parity precision needs fp32 parameters")
            if b.s2d:
                for plane in range(NP):
                    _lib.check(lib.ryolo_space_to_depth(vp(b.src.ptr + 2 * plane * _lo(b.src)), b.src.cs, B, b.src.h, b.src.w,
                                                        b.cin, vp(b.xs.data_ptr() + 2 * plane * b.p4), b.xs.shape[-1], st),
                               "s2d")
                xbase, xcs, xoff, xlo = b.xs.data_ptr(), b.xs.shape[-1], 0, b.p4
            else:
                xbase, xcs, xoff, xlo = b.src.buf.data_ptr(), b.src.cs, b.src.ch_off, _lo(b.src)
            if b.pw_ver != w._version:
                wt = w.detach()
                if b.i == 0:
                    wt = wt.reshape(b.cout, 27, 1, 1)
                _lib.check(lib.ryolo_px_pack_weights(_lib.ptr(wt.contiguous()), b.cout, b.cin_eff, b.k_eff, NTERMS, W_CODE,
                                                     2 if b.s2d else 0, _lib.ptr(b.pw), st), "px_pack_weights")
                b.pw_ver = w._version
            _lib.check(lib.ryolo_px_conv(vp(xbase), xcs, xoff, xlo, b.cin_eff, _lib.ptr(b.pw), NTERMS, A_CODE, B, b.gh, b.gw_,
                                         b.k_eff, b.cout, _lib.ptr(b.z), b.po, b.po, 0, st), "px_conv")
            if b.is_head:
                bias = seq.Conv2d.bias
                _lib.check(lib.ryolo_px_to_nchw(_lib.ptr(b.z), b.po, B, b.cout, b.oh, b.ow,
                                                _lib.ptr(bias.detach()) if bias is not None else None, _lib.ptr(b.out), st),
                           "px_to_nchw")
                continue
            bn = seq.BatchNorm2d
            if self.train:
                _lib.check(lib.ryolo_px_bn_stats(_lib.ptr(b.z), b.po, B, b.oh, b.ow, b.cout, _lib.ptr(b.sums), st), "px_bn_stats")
                bn_counters.append(bn.num_batches_tracked)
            _lib.check(lib.ryolo_px_bn_finalize(_lib.ptr(b.sums), b.cout, float(B * b.oh * b.ow), bn.eps, bn.momentum,
                                                _lib.ptr(bn.weight), _lib.ptr(bn.bias), 0 if self.train else 1,
                                                _lib.ptr(b.mean), _lib.ptr(b.invstd), _lib.ptr(b.scale), _lib.ptr(b.shift),
                                                _lib.ptr(bn.running_mean), _lib.ptr(bn.running_var), st), "px_bn_finalize")
            if b.has_act:
                sw = seq.activation.weight
                if sw.numel() != 1 or sw.dtype != torch.float32:
                    raise NotImplementedError("PReLU with per-channel or non-fp32 slope")
                b.slope_dev = sw.data_ptr()
            else:
                b.slope_dev = None
            _lib.check(lib.ryolo_px_bn_act_fwd(_lib.ptr(b.z), b.po, B, b.oh, b.ow, b.cout, _lib.ptr(b.scale), _lib.ptr(b.shift),
                                               vp(b.slope_dev), vp(b.res.ptr) if b.res is not None else None,
                                               b.res.cs if b.res is not None else 0, _lo(b.res) if b.res is not None else 0,
                                               vp(b.y.ptr), b.y.cs, _lo(b.y), int(b.fuse_up), NP, st), "px_bn_act_fwd")
        if bn_counters:
            with torch.no_grad():
                torch._foreach_add_(bn_counters, 1)
        self.gen += 1
        self.consumed = False
        return [b.out for b in self.heads]

    # ------------------------------------------------------------------------------------------------------
    def backward(self, grads):
        """grads: fp32 [B, na, ny, nx, no] per head (autograd layout).  Returns fresh gradient tensors keyed by
        (block index, 'Module.param')."""
        m, lib, B = self.model, _lib.lib, self.batch
        st = _lib.stream_ptr(self.device)
        vp = ctypes.c_void_p
        pg = {}
        for b, g in zip(self.heads, grads):
            g = g.contiguous().float()
            na, no = g.shape[1], g.shape[4]
            if m.module_list[b.i].Conv2d.bias is not None:
                pg[(b.i, "Conv2d.bias")] = g.double().sum((0, 2, 3)).reshape(-1).float()
            _lib.check(lib.ryolo_px_head_grad(_lib.ptr(g), B, na, no, b.oh, b.ow, _lib.ptr(b.dz), b.dz.shape[-1], b.po, NP, st),
                       "px_head_grad")
        for b in reversed(self.blocks):
            seq = m.module_list[b.i]
            if not b.is_head:
                b.dz.zero_()            # shared scratch: the previous block's data would sit in this block's halo
                _lib.check(lib.ryolo_px_bn_act_bwd(vp(b.gy.ptr), b.gy.cs, int(b.fuse_up), _lib.ptr(b.z), b.po, B, b.oh, b.ow,
                                                   b.cout, _lib.ptr(b.scale), _lib.ptr(b.shift), _lib.ptr(b.mean),
                                                   _lib.ptr(b.invstd), vp(b.slope_dev), 1, _lib.ptr(b.bsums), _lib.ptr(b.dz),
                                                   b.dz.shape[-1], b.po, vp(b.gres.ptr) if b.gres is not None else None,
                                                   b.gres.cs if b.gres is not None else 0, int(b.gres_acc), NP, st), "px_bn_act_bwd")
                f = b.bsums.float()
                pg[(b.i, "BatchNorm2d.bias")] = f[:b.cout]
                pg[(b.i, "BatchNorm2d.weight")] = f[b.cout:2 * b.cout]
                if b.has_act:
                    pg[(b.i, "activation.weight")] = f[2 * b.cout:]
            # ---- weight gradient: segmented wgrad GEMM over all planes of dz and of the source buffer ----
            b.dw.zero_()
            xcs = b.xw_buf.shape[-1]
            _lib.check(lib.ryolo_px_wgrad(_lib.ptr(b.dz), NP * b.po, NP * b.po, _lib.ptr(b.xw_buf), xcs, xcs, B, b.gh, b.gw_,
                                            b.k_eff, _lib.ptr(b.dw), st), "wgrad")
            w = seq.Conv2d.weight
            gw = torch.empty(tuple(w.shape), dtype=torch.float32, device=self.device)
            if b.s2d:
                _lib.check(lib.ryolo_px_unpack_wgrad(_lib.ptr(b.dw), b.po, xcs // NP, NP, 2, b.cout, b.cin, 3, 0, _lib.ptr(gw), st),
                           "px_unpack_wgrad")
            else:
                _lib.check(lib.ryolo_px_unpack_wgrad(_lib.ptr(b.dw), b.po, xcs // NP, NP, 0, b.cout, b.cin, b.k_eff,
                                                     b.src.ch_off, _lib.ptr(gw), st), "px_unpack_wgrad")
            pg[(b.i, "Conv2d.weight")] = gw
            if b.i == 0:
                continue
            # ---- input gradient ----
            _lib.check(lib.ryolo_px_pack_weights(_lib.ptr(w.detach().contiguous()), b.cin_eff, b.cout,
                                                 -2 if b.s2d else b.k_eff, NTERMS, W_CODE, 3 if b.s2d else 1,
                                                 _lib.ptr(b.pwd), st), "px_pack_weights dgrad")
            if b.s2d:
                _lib.check(lib.ryolo_px_conv(_lib.ptr(b.dz), NP * b.po, 0, b.po, b.cout, _lib.ptr(b.pwd), NTERMS, A_CODE, B,
                                             b.gh, b.gw_, -2, b.cin_eff, _lib.ptr(b.dxs), b.p4, b.p4, 0, st), "px dgrad s2d")
                _lib.check(lib.ryolo_px_depth_to_space(_lib.ptr(b.dxs), b.p4, B, b.src.h, b.src.w, b.cin, vp(b.gsrc.ptr),
                                                       b.gsrc.cs, int(b.gsrc_acc), st), "px_d2s")
            else:
                _lib.check(lib.ryolo_px_conv(_lib.ptr(b.dz), NP * b.po, 0, b.po, b.cout, _lib.ptr(b.pwd), NTERMS, A_CODE, B,
                                             b.gh, b.gw_, b.k_eff, b.cin, vp(b.gsrc.ptr), b.gsrc.cs, L.round_up(b.cin, 4),
                                             int(b.gsrc_acc), st), "px dgrad")
        self.consumed = True
        return pg


class DarknetParityFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, plan, x, names, *params):
        # weak, as in DarknetTrainFn: a caller that keeps this step's heads (whose grad_fn is this node) must not keep the
        # plan alive after the model has replaced it
        ctx.plan, ctx.names = weakref.ref(plan), names
        outs = plan.forward(x)
        ctx.gen = plan.gen
        m = plan.model
        res = []
        for b, yi in zip(plan.heads, m.yolo_layers):
            layer = m.module_list[yi]
            if (layer.nx, layer.ny) != (b.ow, b.oh):
                layer.create_grids((plan.h, plan.w), (b.ow, b.oh), plan.device, torch.float32)
            res.append(b.out.view(plan.batch, layer.na, layer.nc + 6, b.oh, b.ow).permute(0, 1, 3, 4, 2).contiguous())
        return tuple(res)

    @staticmethod
    def backward(ctx, *grads):
        plan = ctx.plan()
        if plan is None:
            raise RuntimeError("Darknet parity plan: the plan of this forward was dropped (the model ran another shape or "
                               "mode, or moved) before its backward")
        check_activations(plan, ctx.gen)
        m = plan.model
        gl = []
        for g, b, yi in zip(grads, plan.heads, m.yolo_layers):
            if g is None:        # head not used by the loss
                layer = m.module_list[yi]
                g = torch.zeros((plan.batch, layer.na, b.oh, b.ow, layer.nc + 6), dtype=torch.float32, device=plan.device)
            gl.append(g)
        pg = plan.backward(gl)
        out = []
        for name in ctx.names:
            parts = name.split(".")
            out.append(pg.get((int(parts[1]), parts[2] + "." + parts[3])))
        ddp = getattr(m, "_ddp", None)
        if ddp is not None:
            # data-parallel replicas (parallel.DistributedDataParallel): average the gradients over the ranks.  One flat
            # all-reduce after backward -- this path is the precision reference, not the throughput mode.
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size(ddp["group"]) > 1:
                have = [g for g in out if g is not None]
                flat = torch._utils._flatten_dense_tensors(have)
                dist.all_reduce(flat, group=ddp["group"])
                flat.div_(dist.get_world_size(ddp["group"]))
                it = iter(torch._utils._unflatten_dense_tensors(flat, have))
                out = [next(it) if g is not None else None for g in out]
        return (None, None, None) + tuple(out)
