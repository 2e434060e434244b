"""Training-mode execution of ``Darknet`` on libryolo.so: forward with batch-statistics BatchNorm and the full backward
(reference: train.py:268-282 -- ``pred = model(imgs)``; ``loss.backward()`` through nn.Conv2d / BatchNorm2d / PReLU,
shortcut, route, upsample).

Per conv block:  z = conv(x, W) (wgmma implicit GEMM, raw, bf16)  ->  batch statistics (bn_stats)  ->
y = prelu(z*scale + shift) [+ shortcut] [2x2 replicated] (bn_act_fwd).  Backward, in reverse:  bn_act_bwd (d-gamma,
d-beta, d-slope, dz in place of z, shortcut gradient)  ->  wgrad (wgmma GEMM over pixels)  ->  dgrad (the SAME
implicit-GEMM kernel as forward with the taps mirrored and the weight matrix transposed, accumulating into the
source's gradient buffer through the kernel's residual input).  Stride-2 blocks run their adjoints on the input grid
through a zero-inserted copy of dz.  The first layer (3 channels) goes through an im2col of the image so that it uses
the same kernels.  Activations and activation gradients are bf16 (padded NHWC), parameter gradients fp32.

The whole network is ONE autograd.Function: PyTorch's autograd sees the three head tensors on the outside (so the
loss stays ordinary PyTorch, reference model/loss.py) and receives the parameter gradients in ``parameters()`` order.
Like stock autograd, the backward follows ``requires_grad``: each trainable mask gets a backward schedule of its own
(``Schedule``) that runs only the launches whose results reach a trainable parameter (reference train.py:120-135 and
:215-220 freeze all but the heads, or the backbone)."""
import ctypes
import weakref

import torch

from . import _lib
from . import graph as G
from . import layout as L
from .pool import ActivationPool

_EPS = 1e-5
# the widest head the training backward takes: ryolo_head_grad_nchw_to_padded / ryolo_head_bias_grad reject c > 2048
# (csrc/loss.cu); 72 anchors per head allow up to 22 classes
HEAD_GRAD_MAX_CHANNELS = 2048


class _Block:
    pass


class TrainPlan:
    """The training step at one (batch, height, width).  Its shape-sized storage comes from `pool` (the model's training
    ActivationPool, shared with the plans of its other shapes; None: zeroed tensors of its own), its parameter-sized
    device state -- packed weights, gradient arena, split-K weight-gradient arena, all-reduce buckets -- from `shared`, a
    dict the model keeps once for the plans of every shape.

    Every zero-initialised buffer is either rewritten by every step before it is read, or restored by the pool when the
    plan takes the storage over (``ActivationPool.padded``: the halo and the channels no kernel writes); each
    allocation below says which."""

    def __init__(self, model, batch, height, width, device, pool=None, shared=None):
        self.model, self.batch, self.h, self.w, self.device = model, batch, height, width, device
        self.pool = pool if pool is not None else ActivationPool(device)
        self.shared = shared if shared is not None else {}
        self.halo = None             # the pool's restore table of this plan (set by the model)
        P = self.pool
        g = G.Graph(model, height, width, ("se", "d-convolutional"), "block type %r has no training kernel")
        if not model.yolo_layers and any(cv.is_head for cv in g.convs.values()):
            # the head bookkeeping (create_grids, the gradients autograd hands back) zips the heads with yolo_layers
            raise NotImplementedError("training needs the YOLO layers of the graph; YOLO-less trunks run in eval only")
        wide = [(i, cv.cout) for i, cv in sorted(g.convs.items()) if cv.is_head and cv.cout > HEAD_GRAD_MAX_CHANNELS]
        if wide:
            # refused here, before any launch: the head cotangent's transpose would reject it in the middle of a backward
            raise NotImplementedError("training heads are limited to %d channels (ryolo_head_grad_nchw_to_padded); "
                                      "head conv(s) %s have more (anchors per head * (classes + 6)); such a model "
                                      "runs in eval only" % (HEAD_GRAD_MAX_CHANNELS, wide))
        # activation buffers (y) and their gradient twins; concat groups share one buffer.  Interior real channels: the
        # producer (y) / the first backward writer (gy) writes them every step; halo and padding channels are restored
        bufs = G.Buffers(g, lambda hh, ww, cs: (P.padded(batch, hh, ww, cs, None), P.padded(batch, hh, ww, cs, None)), 32)

        # first layer input: im2col of the image (27 real channels in a 64-channel padded NHWC buffer); restored beyond 27
        self.col = P.padded(batch, height, width, 64, 27)
        blocks = []
        self.phase = {}          # (role, shape) -> phase-layout scratch of the dilated convs (blocks run one at a time)
        for t, i in g.ops:
            if t in ("convolutional", "d-convolutional"):
                blk = g.convs[i]
                if i == 0:
                    if not (blk.k == 3 and blk.stride == 1):
                        raise NotImplementedError("first layer must be 3x3 stride 1")
                    blk.src = G.View(self.col, 0, 27, height, width)
                    blk.gsrc = None
                    blk.k_eff = 1                       # runs as a 1x1 conv over the im2col buffer
                else:
                    blk.src, blk.gsrc = bufs.view(i - 1), bufs.gview(i - 1)
                    blk.k_eff = blk.k
                blk.se = None
                bn_ = 256 if blk.cout > 128 else (128 if blk.cout > 64 else 64)
                blk.cout_pad = L.round_up(blk.cout, bn_)     # GEMM tile extent (weights / dW)
                blk.zcs = L.round_up(blk.cout, 32)           # channel stride of z / dz (TMA zero-fills up to the tile)
                blk.cin = blk.src.c
                blk.cin_pad = L.round_up(blk.cin, 64)
                if blk.is_head:
                    # fp32 NCHW head output: every element written by the head conv every step
                    blk.out = P.take((batch, blk.cout, blk.oh, blk.ow), torch.float32)
                    # gradient of the head output: ryolo_head_grad_nchw_to_padded writes channels < cout; rest restored
                    blk.dz = P.padded(batch, blk.oh, blk.ow, blk.zcs, blk.cout)
                    blk.res = blk.gres = None
                else:
                    # raw conv output / dz: the conv (or the weight_from block's bn_act_bwd) writes channels < cout
                    blk.z = P.padded(batch, blk.oh, blk.ow, blk.zcs, blk.cout)
                    blk.y, blk.gy = bufs.out(blk.mat)
                    if blk.fuse_res:
                        blk.res, blk.gres = bufs.view(blk.shortcut), bufs.gview(blk.shortcut)
                    else:
                        blk.res = blk.gres = None
                    blk.sums = torch.zeros(2 * blk.cout + 1, dtype=torch.float32, device=device)
                    blk.mean, blk.invstd, blk.scale, blk.shift = (torch.zeros(blk.cout, dtype=torch.float32, device=device)
                                                                  for _ in range(4))
                blk.s2d = i > 0 and blk.s2d
                if blk.s2d:
                    # 3x3/stride-2 block on the space-to-depth copy of its input: 2x2 taps, 4C channels, stride 1
                    blk.xs_cs = L.round_up(4 * blk.src.c, 64)
                    # space-to-depth input and its dgrad output: channels < 4C written every step, the rest restored
                    blk.xs = P.padded(batch, blk.src.h // 2, blk.src.w // 2, blk.xs_cs, 4 * blk.src.c)
                    blk.dxs = P.padded(batch, blk.src.h // 2, blk.src.w // 2, blk.xs_cs, 4 * blk.src.c)
                    blk.k_eff = 2
                    blk.cin_eff, blk.cin_pad = 4 * blk.src.c, blk.xs_cs
                    blk.fdesc = L.make_desc(batch, blk.src.h // 2, blk.src.w // 2, blk.cin_eff, blk.xs_cs, blk.cout,
                                            0 if blk.is_head else blk.zcs, 2, 1, False, 0.0, False, 0, False, blk.is_head)
                    blk.ddesc = L.make_desc(batch, blk.src.h // 2, blk.src.w // 2, blk.cout, blk.zcs, blk.cin_eff,
                                            blk.xs_cs, -2, 1, False, 0.0, False, 0, False, False)
                else:
                    blk.cin_eff = blk.cin
                    if blk.stride == 2:
                        # zero-inserted dz: ryolo_zero_insert2x writes the even pixels only, the whole buffer is restored
                        blk.dz_up = P.padded(batch, blk.src.h, blk.src.w, blk.zcs, 0)
                    # forward descriptor: raw conv (no bias / activation); heads keep their bias and write fp32 NCHW
                    blk.fdesc = L.make_desc(batch, blk.src.h, blk.src.w, blk.cin, blk.src.cs, blk.cout,
                                            0 if blk.is_head else blk.zcs, blk.k_eff, blk.stride, False, 0.0, False, 0,
                                            False, blk.is_head)
                    if i > 0:
                        # dgrad: stride-1 conv of dz (at the INPUT resolution) with mirrored taps / transposed weights
                        blk.ddesc = L.make_desc(batch, blk.src.h, blk.src.w, blk.cout, blk.zcs, blk.cin, blk.gsrc.cs,
                                                blk.k, 1, False, 0.0, False, blk.gsrc.cs, False, False)
                if blk.owner is not None:
                    self._linear_block(blk, batch, device)
                blk.dw_shape = (blk.k_eff * blk.k_eff, blk.cout_pad, blk.cin_pad)
                if blk.owner is not None:
                    blocks.append(blk)           # shares the owner's pw / pwd / dw (set below)
                    continue
                # packed weight operands: repacked by every forward (_pack_all), shared by the plans of every shape
                blk.pw = self._shared_bytes(("pw", i), _lib.lib.ryolo_conv_packed_weight_bytes(ctypes.byref(blk.fdesc)))
                if i > 0:
                    blk.pwd = self._shared_bytes(("pwd", i),
                                                 _lib.lib.ryolo_conv_packed_weight_bytes(ctypes.byref(blk.ddesc)))
                blocks.append(blk)
            else:
                # out of place: u = x * s gets a buffer pair of its own and views[i]; views[i - 1] stays x, so that the
                # shortcut three blocks later (`from=-4`) and concat routes read the unscaled tensor like the reference.
                # The SE runs with the block that produced x: forward after its bn_act_fwd, backward before its bn_act_bwd.
                x, gx = bufs.view(i - 1), bufs.gview(i - 1)
                prod = [p_ for p_ in blocks if not p_.is_head and p_.y is x]
                if len(prod) != 1 or prod[0].se is not None or x.c != int(g.defs[i]["channels"]):
                    raise NotImplementedError("[se] at block %d does not follow a conv block's output" % i)
                se = _Block()
                se.i, se.x, se.gx, se.c, se.h, se.w = i, x, gx, x.c, x.h, x.w
                se.cr = model.module_list[i].fc[0].weight.shape[0]
                se.u, se.gu = bufs.out(i)
                # SE scratch: outputs of ryolo_se_fwd (m, p, s) and ryolo_se_bwd (ds, dm), written every step
                se.m, se.s, se.ds, se.dm = (P.take((batch * x.c,), torch.float32) for _ in range(4))
                se.p = P.take((batch * se.cr,), torch.float32)
                prod[0].se = se
        self.blocks = blocks
        P.channels(bufs.channels)
        by_index = {b.i: b for b in blocks}
        for b in blocks:
            if b.owner is not None:
                ow = by_index[b.owner]
                if ow.owner is not None or ow.s2d or ow.stride != 1 or ow.k != b.k or ow.cout_pad != b.cout_pad or \
                        ow.cin_pad != b.cin_pad:
                    raise NotImplementedError("block %d: weight_from=%d has a different training geometry" % (b.i, b.owner))
                b.owner_blk = ow
                b.pw, b.pwd = ow.pw, ow.pwd
        # a bias (+ PReLU) conv without BatchNorm runs bn_act_fwd / bn_act_bwd with fixed statistics: scale 1, shift =
        # the conv bias (mean 0, invstd 1 are never read with has_bn = 0); d-beta is the bias gradient
        for b in blocks:
            if not b.is_head and b.owner is None and not b.has_bn:
                b.scale.fill_(1.0)
                b.invstd.fill_(1.0)
        self.scratch_sums = torch.zeros(2 * 2048 + 1, dtype=torch.float32, device=device)
        ses = [b.se for b in blocks if b.se is not None]
        # SE workspace: written before it is read within each launch
        self.se_ws = P.take((max([_lib.lib.ryolo_se_workspace_bytes(batch, se.h, se.w, se.c, se.cr) for se in ses] + [0]),),
                            torch.uint8)
        # a block whose output feeds a space-to-depth (3x3 / stride 2) block writes the s2d copy itself (bn_act_fwd_s2d)
        for c_ in blocks:
            c_.xs_from_producer = False
        for c_ in blocks:
            if c_.s2d:
                prod = [p_ for p_ in blocks if not p_.is_head and p_.y is c_.src and not p_.fuse_up and p_.owner is None]
                if len(prod) == 1:
                    prod[0].xs_out = c_.xs
                    c_.xs_from_producer = True
        self.zero_bias = torch.zeros(2048, dtype=torch.float32, device=device)
        # static accumulate flags for the backward writers (first writer of a gradient range overwrites)
        written = {}
        for blk in reversed(blocks):
            if blk.se is not None:
                blk.se.gx_acc = G.claim(written, blk.se.gx)
            blk.gres_acc = G.claim(written, blk.gres) if blk.gres is not None else False
            blk.gsrc_acc = G.claim(written, blk.gsrc) if blk.gsrc is not None else False
        # A producer whose output gradient has ONE writer -- the depth_to_space of its space-to-depth consumer -- reads that
        # gradient straight from the consumer's dgrad output (bn_act_bwd mode 2): no d2s pass, no gy buffer traffic.
        for c_ in blocks:
            c_.dxs_direct = False
        for c_ in blocks:
            if not c_.s2d or c_.gsrc is None:
                continue
            key = id(c_.gsrc.buf)
            lo, hi = c_.gsrc.ch_off, c_.gsrc.ch_off + c_.gsrc.c
            writers = [r for r in written.get(key, []) if not (r[1] <= lo or hi <= r[0])]
            prod = [p_ for p_ in blocks if not p_.is_head and p_.gy is c_.gsrc and not p_.fuse_up and p_.owner is None]
            if len(writers) == 1 and len(prod) == 1:
                prod[0].dy_s2d = c_
                c_.dxs_direct = True
        self._build_arena()
        # split-K partial sums of every layer's weight gradient in ONE buffer: one fill per step instead of 75
        # (a weight_from block's wgrad adds into its owner's slot: the owner's gradient sums every use, in backward order)
        off = 0
        for blk in blocks:
            if blk.owner is None:
                blk.dw_off = off
                off += L.round_up(blk.dw_shape[0] * blk.dw_shape[1] * blk.dw_shape[2], 64)
        # its used ranges are zeroed at the start of every backward (_backward_segment)
        self.dw_arena = self._shared_zeros("dw_arena", off)
        for blk in blocks:
            if blk.owner is None:
                n_ = blk.dw_shape[0] * blk.dw_shape[1] * blk.dw_shape[2]
                blk.dw = self.dw_arena[blk.dw_off:blk.dw_off + n_].view(blk.dw_shape)
        for blk in blocks:
            if blk.owner is not None:
                blk.dw = blk.owner_blk.dw
        self._key_now = None
        self.schedules = {}          # trainable mask -> Schedule
        self.sched = self._schedule((True,) * len(self.names))
        self.graphs = None           # CUDA graphs of forward / backward segments (model.use_cuda_graph)
        self.replayed_kernels = 0    # kernels of this library executed through CUDA-graph replays (bench.py gpu_launches)
        self.time_comm = False       # bench.py: record events around the wait for the all-reduces (exposed time)
        self._comm_ev = None

    def _build_arena(self):
        """All parameter gradients live in ONE flat fp32 arena, laid out in the order backward produces them (last block
        first): per block [conv weight | BN (d beta, d gamma) + PReLU d slope] (heads: [weight | bias]).  The kernels write
        straight into it; contiguous ranges of it are the all-reduce buckets (parallel.GradBuckets) and autograd receives
        views of a fresh scaled copy (never of plan-owned memory: AccumulateGrad may keep what it is given)."""
        m = self.model
        off = 0
        self.param_slots = {}        # (block index, "Module.param") -> (offset, numel, shape)
        self.pieces = []             # (lo, hi, slot keys): the arena cut into the units a trainable mask keeps or drops
        bounds = []
        for blk in reversed(self.blocks):
            seq = m.module_list[blk.i]
            if blk.owner is not None:
                # the reference never uses a weight_from block's own Conv2d / BatchNorm2d (nor a d-conv's BatchNorm2d):
                # no slot, autograd receives None for them
                blk.arena_end = None
                continue
            if blk.se is not None:         # the SE's backward runs first in this block's backward
                se = blk.se
                n = se.c * se.cr
                se.gw1_off, se.gw2_off = off, off + L.round_up(n, 4)
                self.param_slots[(se.i, "fc.0.weight")] = (se.gw1_off, n, (se.cr, se.c))
                self.param_slots[(se.i, "fc.2.weight")] = (se.gw2_off, n, (se.c, se.cr))
                off += 2 * L.round_up(n, 4)
                self.pieces.append((se.gw1_off, off, [(se.i, "fc.0.weight"), (se.i, "fc.2.weight")]))
            wshape = tuple(seq.Conv2d.weight.shape)
            n = seq.Conv2d.weight.numel()
            blk.gw_off = off
            self.param_slots[(blk.i, "Conv2d.weight")] = (off, n, wshape)
            off += L.round_up(n, 4)
            self.pieces.append((blk.gw_off, off, [(blk.i, "Conv2d.weight")]))
            if blk.is_head:
                if seq.Conv2d.bias is not None:
                    blk.gb_off = off
                    self.param_slots[(blk.i, "Conv2d.bias")] = (off, blk.cout, (blk.cout,))
                    off += L.round_up(blk.cout, 4)
                    self.pieces.append((blk.gb_off, off, [(blk.i, "Conv2d.bias")]))
            else:
                blk.bs_off = off
                if blk.has_bn:
                    self.param_slots[(blk.i, "BatchNorm2d.bias")] = (off, blk.cout, (blk.cout,))
                    self.param_slots[(blk.i, "BatchNorm2d.weight")] = (off + blk.cout, blk.cout, (blk.cout,))
                elif seq.Conv2d.bias is not None:
                    self.param_slots[(blk.i, "Conv2d.bias")] = (off, blk.cout, (blk.cout,))
                if blk.has_act:
                    self.param_slots[(blk.i, "activation.weight")] = (off + 2 * blk.cout, 1, (1,))
                off += L.round_up(2 * blk.cout + 1, 4)
                self.pieces.append((blk.bs_off, off, [k for k in ((blk.i, "BatchNorm2d.bias"), (blk.i, "BatchNorm2d.weight"),
                                                                  (blk.i, "Conv2d.bias"), (blk.i, "activation.weight"))
                                                      if k in self.param_slots]))
            bounds.append(off)
            blk.arena_end = off
        # every gradient the backward hands out is written by that backward before it is copied out
        self.garena = self._shared_zeros("garena", off)
        for blk in self.blocks:
            if blk.owner is not None:
                continue
            seq = m.module_list[blk.i]
            n = seq.Conv2d.weight.numel()
            blk.gw = self.garena[blk.gw_off:blk.gw_off + n].view(tuple(seq.Conv2d.weight.shape))
            if not blk.is_head:
                blk.bsums = self.garena[blk.bs_off:blk.bs_off + 2 * blk.cout + 1]
            if blk.se is not None:
                se, n = blk.se, blk.se.c * blk.se.cr
                se.gw1 = self.garena[se.gw1_off:se.gw1_off + n]
                se.gw2 = self.garena[se.gw2_off:se.gw2_off + n]
        self.bounds = bounds
        self.names = [nm for nm, _ in m.named_parameters()]

    def _shared_bytes(self, key, nbytes):
        """parameter-sized uint8 device state of the model, one per (key, size) for the plans of every shape"""
        k = key + (nbytes,)
        if k not in self.shared:
            self.shared[k] = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self.shared[k]

    def _shared_zeros(self, key, n):
        k = (key, n)
        if k not in self.shared:
            self.shared[k] = torch.zeros(n, dtype=torch.float32, device=self.device)
        return self.shared[k]

    @property
    def buckets(self):
        """the all-reduce buckets of the current step's schedule (None without DDP)"""
        return self.sched.buckets

    @property
    def segments(self):
        return self.sched.segments

    def _schedule(self, mask):
        """the Schedule of `mask` (requires_grad of every parameter, in parameters() order), derived once and cached:
        changing requires_grad between steps selects another schedule and rebuilds nothing else"""
        sch = self.schedules.get(mask)
        if sch is None:
            sch = self.schedules[mask] = Schedule(self, mask)
        return sch

    # ------------------------------------------------------------------------------------------------------
    def _slopes(self):
        # PReLU slopes stay on the device (kernels read nn.PReLU.weight through slope_dev): no host synchronisation
        m = self.model
        for b in self.blocks:
            if b.has_act:
                wgt = m.module_list[b.i].activation.weight
                if wgt.numel() != 1 or wgt.dtype != torch.float32:
                    raise NotImplementedError("PReLU with per-channel or non-fp32 slope")
                b.slope_dev = wgt.data_ptr()
            else:
                b.slope_dev = None
            b.slope = 1.0

    def _param_key(self):
        """storage identity of everything the captured graphs point at"""
        return tuple(p.data_ptr() for p in self.model.parameters()) + tuple(b.data_ptr() for b in self.model.buffers())

    # ---- multi-tensor pack / unpack (csrc/multi.cu): job tables in device memory, rebuilt when parameter storage moves ----
    def _job_table(self, jobs, cls):
        if not jobs:
            return None, None, 0, 0
        arr = (cls * len(jobs))(*jobs)
        raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self.device)
        sizes = []
        for j in jobs:
            if cls is _lib.PackJob:
                sizes.append(j.ks * j.ks * j.cout_pad * j.cin_pad)
            else:
                sizes.append(j.cout * j.cin * j.ks * j.ks)
        prefix = torch.tensor([0] + list(torch.tensor(sizes, dtype=torch.int64).cumsum(0).tolist()), dtype=torch.int64)
        return raw, prefix.to(self.device), len(jobs), int(prefix[-1])

    def _multi_tables(self):
        key = self._key_now if self._key_now is not None else self._param_key()
        sch = self.sched
        if sch.multi is not None and sch.multi["key"] == key:
            return sch.multi
        m = self.model

        def pads(cout, cin):
            bn_ = 256 if cout > 128 else (128 if cout > 64 else 64)
            return L.round_up(cout, bn_), L.round_up(cin, 64)
        pack = []
        for blk in self.blocks:
            if blk.owner is not None:
                continue
            w = m.module_list[blk.i].Conv2d.weight
            if blk.i == 0:
                cout, cin, ks, mode = blk.cout, 27, 1, 0                       # im2col form: [cout, 27, 1, 1]
            elif blk.s2d:
                cout, cin, ks, mode = blk.cout, blk.cin_eff, 2, 2
            else:
                cout, cin, ks, mode = blk.cout, blk.cin, blk.k_eff, 0
            cp, kp = pads(cout, cin)
            assert blk.pw.numel() == ks * ks * cp * kp * 2, (blk.i, blk.pw.numel(), ks, cp, kp)
            pack.append(_lib.PackJob(w.data_ptr(), blk.pw.data_ptr(), cout, cin, ks, cp, kp, mode))
            if blk.i in sch.pwd_used:                                            # dgrad operand: mirrored taps, transposed
                if blk.s2d:
                    cout_d, cin_d, ks_d, mode_d = blk.cin_eff, blk.cout, 2, 3
                else:
                    cout_d, cin_d, ks_d, mode_d = blk.cin, blk.cout, blk.k, 1
                cpd, kpd = pads(cout_d, cin_d)
                assert blk.pwd.numel() == ks_d * ks_d * cpd * kpd * 2, (blk.i, blk.pwd.numel(), ks_d, cpd, kpd)
                pack.append(_lib.PackJob(w.data_ptr(), blk.pwd.data_ptr(), cout_d, cin_d, ks_d, cpd, kpd, mode_d))
        unpack = []
        for seg in sch.segments:
            jobs = []
            for blk in seg:
                if blk.owner is not None or "wgrad" not in sch.run[blk.i]:
                    continue
                if blk.s2d:
                    jobs.append(_lib.UnpackJob(blk.dw.data_ptr(), blk.gw.data_ptr(), blk.cout_pad, blk.cin_pad, 2, blk.cout,
                                               blk.src.c, 3))
                else:
                    jobs.append(_lib.UnpackJob(blk.dw.data_ptr(), blk.gw.data_ptr(), blk.cout_pad, blk.cin_pad, 0, blk.cout,
                                               blk.cin, blk.k_eff))
            unpack.append(self._job_table(jobs, _lib.UnpackJob))
        sch.multi = {"key": key, "pack": self._job_table(pack, _lib.PackJob), "unpack": unpack}
        return sch.multi

    def _pack_all(self):
        """every forward and every running dgrad's weight operand of the step in one launch (the weights are constant
        within a step)"""
        for b in self.blocks:
            if b.owner is None and self.model.module_list[b.i].Conv2d.weight.dtype != torch.float32:
                raise RuntimeError("fp32 parameters required")
        raw, prefix, n, total = self._multi_tables()["pack"]
        _lib.check(_lib.lib.ryolo_conv_pack_weights_multi(_lib.ptr(raw), n, _lib.ptr(prefix), total, _lib.stream_ptr(self.device)),
                   "pack_weights_multi")

    def _backward_segment(self, si):
        if si == 0:
            for lo, hi in self.sched.dw_ranges:
                self.dw_arena[lo:hi].zero_()
        for blk in self.sched.segments[si]:
            self._backward_block(blk)
        raw, prefix, n, total = self._multi_tables()["unpack"][si]
        if n:
            _lib.check(_lib.lib.ryolo_conv_unpack_wgrad_multi(_lib.ptr(raw), n, _lib.ptr(prefix), total,
                                                              _lib.stream_ptr(self.device)), "unpack_wgrad_multi")

    def _forward_body(self, x):
        m = self.model
        if any(p.dtype != torch.float32 for p in m.parameters()):
            # .half() models are supported in eval mode (weights are re-packed to bf16 anyway); the fused training step
            # reads and updates fp32 master parameters in place, like apex O1 keeps them (train.py:165-166)
            raise RuntimeError("Darknet training step needs fp32 parameters (call .float(); .half() is an inference option)")
        lib = _lib.lib
        st = _lib.stream_ptr(self.device)
        _lib.check(lib.ryolo_im2col_first(_lib.ptr(x), self.batch, self.h, self.w, _lib.ptr(self.col), st), "im2col")
        n_per_pixel = float(self.batch)
        self._slopes()
        self._pack_all()
        bn_counters = []
        for blk in self.blocks:
            seq = m.module_list[blk.i]
            if blk.owner is not None and not blk.is_head:
                self._linear_fwd(blk, st)
                continue
            x_ptr = blk.src.ptr
            if blk.s2d:
                if not blk.xs_from_producer:
                    _lib.check(lib.ryolo_space_to_depth(ctypes.c_void_p(blk.src.ptr), blk.src.cs, self.batch, blk.src.h,
                                                        blk.src.w, blk.src.c, _lib.ptr(blk.xs), blk.xs_cs, st), "s2d")
                x_ptr = blk.xs.data_ptr()
            if blk.is_head:
                if getattr(blk, "bias_pad", None) is None:
                    blk.bias_pad = L.padded_bias(blk.fdesc, torch.zeros(blk.cout, device=self.device))
                if seq.Conv2d.bias is not None and blk.owner is None:     # a weight_from head runs without bias
                    blk.bias_pad[:blk.cout].copy_(seq.Conv2d.bias.detach())
                _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.fdesc), ctypes.c_void_p(x_ptr), _lib.ptr(blk.pw),
                                                     _lib.ptr(blk.bias_pad), None, _lib.ptr(blk.out), st), "conv head")
                continue
            _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.fdesc), ctypes.c_void_p(x_ptr), _lib.ptr(blk.pw),
                                                 _lib.ptr(self.zero_bias), None, _lib.ptr(blk.z), st), "conv")
            cnt = n_per_pixel * blk.oh * blk.ow
            if blk.has_bn:
                bn = seq.BatchNorm2d
                _lib.check(lib.ryolo_bn_stats_finalize(_lib.ptr(blk.z), blk.zcs, self.batch, blk.oh, blk.ow, blk.cout,
                                                       _lib.ptr(blk.sums), bn.eps, bn.momentum, _lib.ptr(bn.weight),
                                                       _lib.ptr(bn.bias), _lib.ptr(blk.mean), _lib.ptr(blk.invstd),
                                                       _lib.ptr(blk.scale), _lib.ptr(blk.shift), _lib.ptr(bn.running_mean),
                                                       _lib.ptr(bn.running_var), st), "bn_stats_finalize")
                bn_counters.append(bn.num_batches_tracked)
            elif seq.Conv2d.bias is not None:
                blk.shift.copy_(seq.Conv2d.bias.detach())
            xs_out = getattr(blk, "xs_out", None)
            if xs_out is not None:
                _lib.check(lib.ryolo_bn_act_fwd_s2d(_lib.ptr(blk.z), blk.zcs, self.batch, blk.oh, blk.ow, blk.cout,
                                                    _lib.ptr(blk.scale), _lib.ptr(blk.shift), blk.slope, int(blk.has_act),
                                                    ctypes.c_void_p(blk.res.ptr) if blk.res is not None else None,
                                                    blk.res.cs if blk.res is not None else 0, ctypes.c_void_p(blk.y.ptr),
                                                    blk.y.cs, ctypes.c_void_p(blk.slope_dev), _lib.ptr(xs_out),
                                                    xs_out.shape[-1], st), "bn_act_fwd_s2d")
            else:
                _lib.check(lib.ryolo_bn_act_fwd(_lib.ptr(blk.z), blk.zcs, self.batch, blk.oh, blk.ow, blk.cout,
                                                _lib.ptr(blk.scale), _lib.ptr(blk.shift), blk.slope, int(blk.has_act),
                                                ctypes.c_void_p(blk.res.ptr) if blk.res is not None else None,
                                                blk.res.cs if blk.res is not None else 0, ctypes.c_void_p(blk.y.ptr),
                                                blk.y.cs, int(blk.fuse_up), ctypes.c_void_p(blk.slope_dev), st), "bn_act_fwd")
            if blk.se is not None:
                self._se_fwd(blk.se, st)
        if bn_counters:
            with torch.no_grad():
                torch._foreach_add_(bn_counters, 1)
        # the fp32 NCHW buffers the head convolutions wrote; DarknetTrainFn's caller hands out permuted VIEWS of them
        # ([B, na, ny, nx, no] like model/models.py:190-192, without the .contiguous() copy of 0.5 GB per step)
        return [blk.out for blk in self.heads]

    def forward(self, x, mask=None):
        """mask: requires_grad of every parameter in parameters() order (None: all); selects the backward schedule"""
        m = self.model
        self.sched = self._schedule(tuple(mask) if mask is not None else (True,) * len(self.names))
        self.heads = [b for b in self.blocks if b.is_head]
        for blk, yi in zip(self.heads, m.yolo_layers):
            layer = m.module_list[yi]
            if (layer.nx, layer.ny) != (blk.ow, blk.oh):
                layer.create_grids((self.h, self.w), (blk.ow, blk.oh), self.device, torch.float32)
        self._key_now = self._param_key()      # once per step: storage identity of parameters / buffers
        if self.halo is not None:              # the pool served another plan since this plan's last step
            self.pool.activate(self.halo, _lib.stream_ptr(self.device))
        if getattr(m, "use_cuda_graph", False):
            outs = self._forward_graph(x)
        else:
            outs = self._forward_body(x)
        self.pool.gen += 1
        self.pool.consumed = False
        return outs

    # ---- CUDA-graph form (opt-in, model.use_cuda_graph): the ~1100 launches of a forward and the ~1300 of a backward are
    # replayed as a handful of graphs -- what makes the step launch-bound at small per-GPU batches (8 GPUs: 8 images per
    # rank) is the host, not the GPU.  Inputs are copied into static buffers; outputs are static buffers that the next
    # step overwrites (standard CUDA-graph semantics).
    def _forward_graph(self, x):
        key = (self._key_now, self.sched.mask)     # the pack table and the backward segments depend on the schedule
        if self.graphs is None or self.graphs["key"] != key:
            self.graphs = {"key": key, "pool": None}
            self.x_static = x.clone()          # outside the pool: only plans that capture need it
            eager = self._forward_body(self.x_static)         # this call's forward, eagerly (also the capture warm-up)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            c0 = _lib.lib.ryolo_launch_count()
            with torch.cuda.graph(g):
                outs = self._forward_body(self.x_static)      # captured, not executed
            self.graphs["pool"] = g.pool()
            self.graphs["fwd"] = (g, outs)
            self.graphs["fwd_kernels"] = int(_lib.lib.ryolo_launch_count() - c0)   # this library's kernels in the graph
            return eager
        g, outs = self.graphs["fwd"]
        self.x_static.copy_(x)
        g.replay()
        self.replayed_kernels += self.graphs["fwd_kernels"]
        return outs

    # ------------------------------------------------------------------------------------------------------
    def _head_grads(self, grads):
        """autograd's head cotangents, fp32 NCHW [B, na*no, ny, nx] (the layout of the head buffers; contiguous without a
        copy when the consumer differentiated the permuted view in place, as loss._FusedLoss does) -> bias gradients +
        padded-NHWC bf16 dz of the head convs"""
        lib = _lib.lib
        st = _lib.stream_ptr(self.device)
        for blk, g in zip(self.heads, grads):
            run = self.sched.run[blk.i]
            if not run & {"head", "head_bias"}:
                continue
            g = g.contiguous().float()
            gb = self.garena[blk.gb_off:blk.gb_off + blk.cout] if (blk.i, "Conv2d.bias") in self.param_slots else None
            if gb is not None:       # the bias gradient = per-channel sums of g, taken on the way by the same kernel
                gb.zero_()
            if "head_bias" in run:   # only the bias trains: its sums alone, the same bits
                _lib.check(lib.ryolo_head_bias_grad(_lib.ptr(g), self.batch, blk.cout, blk.oh, blk.ow, _lib.ptr(gb), st),
                           "head_bias_grad")
                continue
            _lib.check(lib.ryolo_head_grad_nchw_to_padded(_lib.ptr(g), self.batch, blk.cout, blk.oh, blk.ow, _lib.ptr(blk.dz),
                                                          blk.zcs, _lib.ptr(gb) if gb is not None else None, st),
                       "head_grad_nchw_to_padded")

    def _se_fwd(self, se, st):
        fc = self.model.module_list[se.i].fc
        _lib.check(_lib.lib.ryolo_se_fwd(ctypes.c_void_p(se.x.ptr), se.x.cs, ctypes.c_void_p(se.u.ptr), se.u.cs, self.batch,
                                         se.h, se.w, se.c, _lib.ptr(fc[0].weight), _lib.ptr(fc[2].weight), se.cr,
                                         _lib.ptr(se.m), _lib.ptr(se.p), _lib.ptr(se.s), _lib.ptr(self.se_ws),
                                         self.se_ws.numel(), st), "se_fwd")

    def _se_bwd(self, se, st):
        fc = self.model.module_list[se.i].fc
        _lib.check(_lib.lib.ryolo_se_bwd(ctypes.c_void_p(se.gu.ptr), se.gu.cs, ctypes.c_void_p(se.x.ptr), se.x.cs,
                                         ctypes.c_void_p(se.gx.ptr), se.gx.cs, int(se.gx_acc), self.batch, se.h, se.w,
                                         se.c, _lib.ptr(fc[0].weight), _lib.ptr(fc[2].weight), se.cr, _lib.ptr(se.m),
                                         _lib.ptr(se.p), _lib.ptr(se.s), _lib.ptr(se.ds), _lib.ptr(se.dm),
                                         _lib.ptr(se.gw1), _lib.ptr(se.gw2), _lib.ptr(self.se_ws), self.se_ws.numel(), st),
                   "se_bwd")

    def _backward_block(self, blk):
        m = self.model
        lib = _lib.lib
        st = _lib.stream_ptr(self.device)
        seq = m.module_list[blk.i]
        run = self.sched.run[blk.i]
        if blk.owner is not None and not blk.is_head:
            self._linear_bwd(blk, run, st)
            return
        if blk.is_head:
            dz = blk.dz
        else:
            if "se" in run:
                self._se_bwd(blk.se, st)
            if "bnact" not in run:
                return
            src_c = getattr(blk, "dy_s2d", None)
            dy_ptr, dy_cs, dy_mode = (blk.gy.ptr, blk.gy.cs, int(blk.fuse_up)) if src_c is None else \
                (src_c.dxs.data_ptr(), src_c.xs_cs, 2)
            _lib.check(lib.ryolo_bn_act_bwd(ctypes.c_void_p(dy_ptr), dy_cs, dy_mode, _lib.ptr(blk.z),
                                            blk.zcs, self.batch, blk.oh, blk.ow, blk.cout, _lib.ptr(blk.scale),
                                            _lib.ptr(blk.shift), _lib.ptr(blk.mean), _lib.ptr(blk.invstd), blk.slope,
                                            int(blk.has_act), int(blk.has_bn), _lib.ptr(blk.bsums),
                                            ctypes.c_void_p(blk.gres.ptr) if blk.gres is not None else None,
                                            blk.gres.cs if blk.gres is not None else 0, int(blk.gres_acc),
                                            ctypes.c_void_p(blk.slope_dev), st),
                       "bn_act_bwd")
            dz = blk.z
        wgrad, dgrad = "wgrad" in run, "dgrad" in run
        if blk.s2d:
            if wgrad:
                _lib.check(lib.ryolo_conv_wgrad(_lib.ptr(dz), blk.zcs, blk.cout_pad, _lib.ptr(blk.xs), blk.xs_cs,
                                                blk.cin_pad, self.batch, blk.src.h // 2, blk.src.w // 2, 2, _lib.ptr(blk.dw),
                                                st), "wgrad s2d")
            if dgrad:
                _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.ddesc), _lib.ptr(dz), _lib.ptr(blk.pwd),
                                                     _lib.ptr(self.zero_bias), None, _lib.ptr(blk.dxs), st),
                           "dgrad s2d")
                if not blk.dxs_direct:
                    _lib.check(lib.ryolo_depth_to_space(_lib.ptr(blk.dxs), blk.xs_cs, self.batch, blk.src.h, blk.src.w,
                                                        blk.src.c, ctypes.c_void_p(blk.gsrc.ptr), blk.gsrc.cs,
                                                        int(blk.gsrc_acc), st), "d2s")
            return
        if blk.stride == 2 and (wgrad or dgrad):
            _lib.check(lib.ryolo_zero_insert2x(_lib.ptr(dz), blk.zcs, self.batch, blk.oh, blk.ow, blk.zcs,
                                               _lib.ptr(blk.dz_up), blk.zcs, blk.src.h, blk.src.w, st), "zero_insert")
            dz = blk.dz_up
        if wgrad:
            _lib.check(lib.ryolo_conv_wgrad(_lib.ptr(dz), blk.zcs, blk.cout_pad, ctypes.c_void_p(blk.src.ptr), blk.src.cs,
                                            blk.cin_pad, self.batch, blk.src.h, blk.src.w, blk.k_eff, _lib.ptr(blk.dw), st),
                       "wgrad")
        if dgrad:
            gp = blk.gsrc.ptr
            blk.ddesc.has_residual = int(blk.gsrc_acc)
            _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.ddesc), _lib.ptr(dz), _lib.ptr(blk.pwd),
                                                 _lib.ptr(self.zero_bias), ctypes.c_void_p(gp) if blk.gsrc_acc else None,
                                                 ctypes.c_void_p(gp), st), "dgrad")

    # ---- weight_from blocks (reference models.py:255-265): a linear conv with the owner's weight, no bias / BN / activation.
    # The forward writes y directly (the conv epilogue, or for a dilated conv the merge, adds the shortcut that follows).
    # The backward takes dz = dy (and d-shortcut += dy) through bn_act_bwd with has_bn = has_act = 0, then the wgrad adds
    # into the owner's dw and the dgrad runs on the owner's pwd.  A dilated 3x3 conv (dh, dw) is an ordinary 3x3 conv on
    # the dh*dw phase images of its input (ryolo_dilate_split); the merge is the split's adjoint, so the backward splits
    # dz, runs wgrad / dgrad on the phase images and merges dx into the source gradient.
    def _phase_buf(self, role, nb, h, w, cs, blk_c):
        key = (role, nb, h, w, cs)
        if key not in self.phase:
            # z / dx phase images: the split / the dgrad writes channels < the real count, the rest is restored
            self.phase[key] = self.pool.padded(nb, h, w, cs, blk_c)
        return self.phase[key]

    def _linear_block(self, blk, batch, device):
        if blk.fuse_up or blk.se is not None:
            raise NotImplementedError("weight_from block %d feeding an upsample or an SE" % blk.i)
        if blk.is_head:
            return
        # blk.z holds dz only: the forward writes y directly
        if blk.dil is None:
            blk.fdesc = L.make_desc(batch, blk.src.h, blk.src.w, blk.cin, blk.src.cs, blk.cout, blk.y.cs, blk.k, 1, False,
                                    0.0, blk.res is not None, blk.res.cs if blk.res is not None else 0, False, False)
            return
        dh, dw = blk.dil
        blk.nb, blk.hp, blk.wp = batch * dh * dw, -(-blk.src.h // dh), -(-blk.src.w // dw)
        # kept for the wgrad; the split writes channels < cin of the interior (zero fill included), the rest is restored
        blk.xp = self.pool.padded(blk.nb, blk.hp, blk.wp, blk.cin_pad, blk.cin)
        blk.zp = self._phase_buf("z", blk.nb, blk.hp, blk.wp, blk.zcs, blk.cout)
        blk.dxp = self._phase_buf("dx", blk.nb, blk.hp, blk.wp, blk.cin_pad, blk.cin)
        blk.fdesc = L.make_desc(blk.nb, blk.hp, blk.wp, blk.cin, blk.cin_pad, blk.cout, blk.zcs, 3, 1, False, 0.0)
        blk.ddesc = L.make_desc(blk.nb, blk.hp, blk.wp, blk.cout, blk.zcs, blk.cin, blk.cin_pad, 3, 1, False, 0.0)

    def _linear_fwd(self, blk, st):
        lib = _lib.lib
        if blk.dil is None:
            _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.fdesc), ctypes.c_void_p(blk.src.ptr), _lib.ptr(blk.pw),
                                                 _lib.ptr(self.zero_bias),
                                                 ctypes.c_void_p(blk.res.ptr) if blk.res is not None else None,
                                                 ctypes.c_void_p(blk.y.ptr), st), "conv (weight_from)")
            return
        dh, dw = blk.dil
        _lib.check(lib.ryolo_dilate_split(ctypes.c_void_p(blk.src.ptr), blk.src.cs, self.batch, blk.src.h, blk.src.w,
                                          blk.cin, dh, dw, _lib.ptr(blk.xp), blk.cin_pad, st), "dilate_split")
        _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.fdesc), _lib.ptr(blk.xp), _lib.ptr(blk.pw),
                                             _lib.ptr(self.zero_bias), None, _lib.ptr(blk.zp), st), "conv (dilated)")
        _lib.check(lib.ryolo_dilate_merge(_lib.ptr(blk.zp), blk.zcs, self.batch, blk.oh, blk.ow, blk.cout, dh, dw,
                                          ctypes.c_void_p(blk.res.ptr) if blk.res is not None else None,
                                          blk.res.cs if blk.res is not None else 0, 0, ctypes.c_void_p(blk.y.ptr), blk.y.cs,
                                          st), "dilate_merge")

    def _linear_bwd(self, blk, run, st):
        lib = _lib.lib
        if "bnact" not in run:
            return
        _lib.check(lib.ryolo_bn_act_bwd(ctypes.c_void_p(blk.gy.ptr), blk.gy.cs, 0, _lib.ptr(blk.z), blk.zcs, self.batch,
                                        blk.oh, blk.ow, blk.cout, _lib.ptr(self.zero_bias), _lib.ptr(self.zero_bias),
                                        _lib.ptr(self.zero_bias), _lib.ptr(self.zero_bias), 0.0, 0, 0,
                                        _lib.ptr(self.scratch_sums),
                                        ctypes.c_void_p(blk.gres.ptr) if blk.gres is not None else None,
                                        blk.gres.cs if blk.gres is not None else 0, int(blk.gres_acc), None, st),
                   "bn_act_bwd (weight_from)")
        wgrad, dgrad = "wgrad" in run, "dgrad" in run
        if blk.dil is None:
            if wgrad:
                _lib.check(lib.ryolo_conv_wgrad(_lib.ptr(blk.z), blk.zcs, blk.cout_pad, ctypes.c_void_p(blk.src.ptr),
                                                blk.src.cs, blk.cin_pad, self.batch, blk.src.h, blk.src.w, blk.k,
                                                _lib.ptr(blk.dw), st), "wgrad (weight_from)")
            if not dgrad:
                return
            gp = blk.gsrc.ptr
            blk.ddesc.has_residual = int(blk.gsrc_acc)
            _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.ddesc), _lib.ptr(blk.z), _lib.ptr(blk.pwd),
                                                 _lib.ptr(self.zero_bias), ctypes.c_void_p(gp) if blk.gsrc_acc else None,
                                                 ctypes.c_void_p(gp), st), "dgrad (weight_from)")
            return
        dh, dw = blk.dil
        if not (wgrad or dgrad):
            return
        _lib.check(lib.ryolo_dilate_split(_lib.ptr(blk.z), blk.zcs, self.batch, blk.oh, blk.ow, blk.cout, dh, dw,
                                          _lib.ptr(blk.zp), blk.zcs, st), "dilate_split (dz)")
        if wgrad:
            _lib.check(lib.ryolo_conv_wgrad(_lib.ptr(blk.zp), blk.zcs, blk.cout_pad, _lib.ptr(blk.xp), blk.cin_pad,
                                            blk.cin_pad, blk.nb, blk.hp, blk.wp, 3, _lib.ptr(blk.dw), st), "wgrad (dilated)")
        if not dgrad:
            return
        _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.ddesc), _lib.ptr(blk.zp), _lib.ptr(blk.pwd),
                                             _lib.ptr(self.zero_bias), None, _lib.ptr(blk.dxp), st),
                   "dgrad (dilated)")
        _lib.check(lib.ryolo_dilate_merge(_lib.ptr(blk.dxp), blk.cin_pad, self.batch, blk.src.h, blk.src.w, blk.cin, dh, dw,
                                          None, 0, int(blk.gsrc_acc), ctypes.c_void_p(blk.gsrc.ptr), blk.gsrc.cs, st),
                   "dilate_merge (dx)")

    def backward(self, grads):
        m = self.model
        overlap = self.buckets is not None and self.buckets.world > 1
        if overlap:
            # leave a few SMs to the NCCL all-reduce kernels that run next to the backward GEMMs (persistent kernels with a
            # static tile schedule would otherwise run a second wave on the SMs NCCL occupies)
            _lib.lib.ryolo_set_reserved_sms(int(getattr(m, "_ddp", {}).get("reserved_sms", 0)))
        try:
            return self._backward(grads)
        finally:
            if overlap:
                _lib.lib.ryolo_set_reserved_sms(0)

    def _backward(self, grads):
        m = self.model
        sch = self.sched
        self._head_grads(grads)
        use_graph = getattr(m, "use_cuda_graph", False) and self.graphs is not None and "fwd" in self.graphs
        if use_graph and "bwd" not in self.graphs:
            # first backward after capture of the forward: run eagerly once (warm-up), then capture every segment
            for si in range(len(sch.segments)):
                self._backward_segment(si)
                if sch.buckets:
                    sch.buckets.ready(sch.ready[si])
            inv = sch.buckets.finish() if sch.buckets else 1.0
            outs = [self.garena[lo:hi] * inv for lo, hi in sch.ranges]
            torch.cuda.synchronize(self.device)
            gs, gk = [], []
            for si in range(len(sch.segments)):
                if not sch.busy[si]:          # nothing to launch: no graph (an empty capture is an error)
                    gs.append(None)
                    gk.append(0)
                    continue
                g = torch.cuda.CUDAGraph()
                c0 = _lib.lib.ryolo_launch_count()
                with torch.cuda.graph(g, pool=self.graphs["pool"]):
                    self._backward_segment(si)
                gs.append(g)
                gk.append(int(_lib.lib.ryolo_launch_count() - c0))
            self.graphs["bwd_kernels"] = gk
            self.graphs["bwd"] = gs
            # the capture passes did not execute; the eager pass above produced this step's gradients
        else:
            for si in range(len(sch.segments)):
                if not use_graph:
                    self._backward_segment(si)
                elif self.graphs["bwd"][si] is not None:
                    self.graphs["bwd"][si].replay()
                    self.replayed_kernels += self.graphs["bwd_kernels"][si]
                if sch.buckets:
                    sch.buckets.ready(sch.ready[si])     # NCCL all-reduce of the finished bucket on the side stream
            if self.time_comm:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
            inv = sch.buckets.finish() if sch.buckets else 1.0
            if self.time_comm:
                e1.record()
                self._comm_ev = (e0, e1)
            # fresh tensors, trainable ranges only: autograd may keep what it is given
            outs = [self.garena[lo:hi] * inv for lo, hi in sch.ranges]
        self.pool.consumed = True
        out = []
        for name in self.names:
            parts = name.split(".")            # module_list.{i}.{Module}.{param} (SE: module_list.{i}.fc.{0|2}.weight)
            key = (int(parts[1]), ".".join(parts[2:]))
            slot = self.param_slots.get(key) if key in sch.trainable else None
            if slot is None:
                out.append(None)
                continue
            r = sch.range_of[key]
            lo = slot[0] - sch.ranges[r][0]
            out.append(outs[r][lo:lo + slot[1]].view(slot[2]))
        return out


class Schedule:
    """The backward of one trainable mask: which launches run, the arena ranges autograd and the all-reduce see, the
    segments and buckets.  Derived over the data edges of the plan (concat views, shortcuts, the fused upsamples, SE
    nodes and weight_from uses):

      up(t)      the tensor t depends on a trainable parameter (a forward walk; a view reads every range it overlaps)
      out(b)     = trainable(b) or up(b.src) or up(b.res): b's output gradient is needed, so bn_act_bwd runs
      se_bwd     iff an fc weight trains or out(b) (its gu is needed)
      wgrad      iff the conv weight trains (a weight_from block: its owner's weight, every use adds into the owner's dw)
      dgrad      iff up(b.src) (with its zero-insert / depth_to_space / dilate merge; split and zero-insert also serve wgrad)
      heads      dz iff the weight trains or up(src); otherwise the bias sums alone when the bias trains

    A gradient range is needed iff up(its tensor): every writer of a needed range then runs, in the order of the full
    plan, so the static accumulate flags stay right.  That is asserted, by the same first-writer walk that set them.  With
    every parameter trainable the schedule is the full plan, launch for launch."""

    def __init__(self, plan, mask):
        if len(mask) != len(plan.names):
            raise ValueError("trainable mask of %d entries for %d parameters" % (len(mask), len(plan.names)))
        self.mask = mask
        self.multi = None        # job tables of the multi-tensor pack / unpack launches (keyed on parameter storage)
        tr = set()
        for name, t in zip(plan.names, mask):
            parts = name.split(".")
            if t:
                tr.add((int(parts[1]), ".".join(parts[2:])))
        self.trainable = tr
        blocks = plan.blocks
        ups = {}                 # buffer id -> [(lo, hi, up)] of the ranges written by the forward so far

        def up(v):
            if v is None or v.buf is None:
                return False
            lo, hi = v.ch_off, v.ch_off + v.c
            return any(u for a, b, u in ups.get(id(v.buf), []) if a < hi and lo < b)

        def record(v, u):
            ups.setdefault(id(v.buf), []).append((v.ch_off, v.ch_off + v.c, u))

        run = self.run = {}
        for b in blocks:
            wi = b.owner if b.owner is not None else b.i
            tw = (wi, "Conv2d.weight") in tr
            up_src = b.i > 0 and up(b.src)
            r = set()
            if b.is_head:
                if tw or up_src:
                    r.add("head")
                elif (b.i, "Conv2d.bias") in tr and (b.i, "Conv2d.bias") in plan.param_slots:
                    r.add("head_bias")
            else:
                tp = b.owner is None and any((b.i, k) in tr for k in ("BatchNorm2d.bias", "BatchNorm2d.weight",
                                                                     "Conv2d.bias", "activation.weight"))
                out = tw or tp or up_src or (b.res is not None and up(b.res))
                if out:
                    r.add("bnact")
                record(b.y, out)
                if b.se is not None:
                    up_u = out or any((b.se.i, k) in tr for k in ("fc.0.weight", "fc.2.weight"))
                    if up_u:
                        r.add("se")
                    record(b.se.u, up_u)
            if tw:
                r.add("wgrad")
            if up_src:
                r.add("dgrad")
            run[b.i] = frozenset(r)

        # the invariant: every writer of a needed gradient range runs, and the first-writer walk over the writers that
        # run gives each of them its full-plan accumulate flag
        written = {}
        for b in reversed(blocks):
            r = run[b.i]
            for kind, v, flag in (("se", b.se.gx if b.se is not None else None, getattr(b.se, "gx_acc", None)),
                                  ("bnact", b.gres, b.gres_acc), ("dgrad", b.gsrc, b.gsrc_acc)):
                if v is None:
                    continue
                assert kind in r or not up(v), ("writer of a needed gradient range pruned", kind, b.i)
                if kind in r:
                    acc = G.claim(written, v)
                    assert acc == flag or not up(v), ("accumulate flag differs from the full plan", kind, b.i)
            p_ = getattr(b, "dy_s2d", None)
            assert p_ is None or "bnact" not in r or "dgrad" in run[p_.i], ("dy read from a pruned dgrad", b.i)
        self.pwd_used = set()        # owners whose packed dgrad operand some running dgrad reads
        for b in blocks:
            if "dgrad" in run[b.i]:
                self.pwd_used.add(b.owner if b.owner is not None else b.i)
        self.dw_ranges = _merge([(b.dw_off, b.dw_off + L.round_up(b.dw.numel(), 64)) for b in blocks
                                 if b.owner is None and "wgrad" in run[b.i]])

        # arena ranges autograd receives and the all-reduce covers: the pieces holding a trainable parameter
        self.ranges = _merge([(lo, hi) for lo, hi, keys in plan.pieces if any(k in tr for k in keys)])
        self.range_of = {}
        for lo, hi, keys in plan.pieces:
            for k in keys:
                if k in tr:
                    self.range_of[k] = next(j for j, (a, b_) in enumerate(self.ranges) if a <= lo and hi <= b_)
        ddp = getattr(plan.model, "_ddp", None)
        from .parallel import GradBuckets
        self.buckets = None
        if ddp:              # one set per mask for the plans of every shape (they share the gradient arena)
            bk = ("buckets", mask, plan.garena.numel())
            if bk not in plan.shared:
                plan.shared[bk] = GradBuckets(plan.garena, plan.bounds, bucket_bytes=ddp["bucket_bytes"],
                                              group=ddp["group"], ranges=self.ranges)
            self.buckets = plan.shared[bk]
        # backward segments = runs of blocks whose gradients complete one bucket (one segment without DDP); ready[s] is
        # the arena offset below which every gradient is final after segment s
        ends = sorted(hi for _, hi in self.buckets.buckets) if self.buckets else []
        segs, cur, self.ready, k = [], [], [], 0
        for b in reversed(blocks):
            cur.append(b)
            if b.arena_end is not None and k < len(ends) and ends[k] <= b.arena_end:
                while k < len(ends) and ends[k] <= b.arena_end:
                    k += 1
                segs.append(cur)
                self.ready.append(b.arena_end)
                cur = []
        if cur:
            segs.append(cur)
            self.ready.append(plan.garena.numel())
        self.segments = segs
        self.busy = [bool((si == 0 and self.dw_ranges) or any(run[b.i] - {"head", "head_bias"} for b in seg))
                     for si, seg in enumerate(segs)]

    def ops(self, plan):
        """the launches of the backward in order, as (kind, layer, accumulate flag or None): what the tests compare"""
        out = []
        for b in plan.blocks:
            if b.is_head:
                out += [(k, b.i, None) for k in ("head", "head_bias") if k in self.run[b.i]]
        for seg in self.segments:
            for b in seg:
                r = self.run[b.i]
                if "se" in r:
                    out.append(("se", b.se.i, b.se.gx_acc))
                if "bnact" in r:
                    out.append(("bnact", b.i, b.gres_acc if b.gres is not None else None))
                if "wgrad" in r:
                    out.append(("wgrad", b.i, None))
                if "dgrad" in r:
                    out.append(("dgrad", b.i, (b.gsrc_acc, b.dxs_direct)))
        return out


def _merge(ranges):
    """sorted, touching ranges joined"""
    out = []
    for lo, hi in sorted(ranges):
        if out and out[-1][1] == lo:
            out[-1] = (out[-1][0], hi)
        else:
            out.append((lo, hi))
    return out


def _comm_wait_ms(self):
    """time the main stream spent waiting for the gradient all-reduces AFTER the last backward kernel was enqueued = the
    exposed (non-overlapped) part of the collective; None when not measured"""
    if self._comm_ev is None:
        return None
    self._comm_ev[1].synchronize()
    return self._comm_ev[0].elapsed_time(self._comm_ev[1])


TrainPlan.last_comm_wait_ms = _comm_wait_ms


def check_activations(plan, gen):
    """the backward of a plan's forward `gen` needs that forward's activations: they live in the plan (not per call), so a
    second forward overwrote them, or a backward already turned z into dz in place.  Stock autograd would handle or
    reject these cases; silently wrong gradients are not an option."""
    if plan.gen != gen or plan.consumed:
        raise RuntimeError("Darknet training plan: the activations of this forward were overwritten by a later forward "
                           "or already consumed by a backward (retain_graph / two forwards before one backward are "
                           "not supported by the fused training path)")


class DarknetTrainFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, plan, x, *params):
        # weak: the head buffers returned below are the plan's own and carry this node as grad_fn, so a strong reference
        # would keep every plan alive (and its pool storage, which growth must free) through that cycle
        ctx.plan = weakref.ref(plan)
        outs = plan.forward(x, ctx.needs_input_grad[2:])
        ctx.gen = plan.pool.gen
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        plan = ctx.plan()
        if plan is None:
            raise RuntimeError("Darknet training plan: the plan of this forward was dropped (a larger shape grew the "
                               "activation pool, or the model moved) before its backward")
        plan.pool.check(ctx.gen)
        gl = []
        for g, blk, yi in zip(grads, plan.heads, plan.model.yolo_layers):
            if g is None:
                g = torch.zeros((plan.batch, blk.cout, blk.oh, blk.ow), dtype=torch.float32, device=plan.device)
            gl.append(g)
        pg = plan.backward(gl)
        return (None, None) + tuple(pg)
