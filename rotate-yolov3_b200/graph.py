"""How Darknet's cfg graph maps to activation buffers and fused conv launches: the one walk over ``module_defs`` that
the eval (models.py), training (train_path.py) and parity-precision (parity_path.py) plans share.  Pure Python over
the parsed cfg and the module tree; the plans allocate their buffers through a callback and do all tensor work.

  * every block's output shape (C, H, W), and the sources of every route;
  * per conv block one launch record (``Conv``): the shortcut or 2x upsample its epilogue absorbs, whether it is a head,
    which layer's output it materialises, whether it may run on a space-to-depth copy of its input;
  * concat placement: the sources of a multi-source route write at their channel offsets of one shared buffer;
  * the first-writer bookkeeping of the backward's gradient ranges.

Refused everywhere, because every plan relies on the layout: a shortcut whose source is not a materialised tensor of the
conv's output shape (the epilogue reads the residual at the output's pixels and channels), and a concat source whose
channel count is not a multiple of 8 (its producer stores at that channel offset through TMA, 16-byte aligned)."""
from . import layout as L
from .parse_config import dilation


def route_sources(d, i):
    """the layer indices the route block ``d`` at index ``i`` reads"""
    return [l if l > 0 else i + l for l in (int(x) for x in d["layers"].split(","))]


class View:
    """a [B, H, W, C] activation at channel ch_off of a (possibly wider) padded-NHWC buffer; buf None: the activation
    exists only in a consumer's space-to-depth buffer"""

    def __init__(self, buf, ch_off, c, h, w):
        self.buf, self.ch_off, self.c, self.h, self.w = buf, ch_off, c, h, w

    @property
    def cs(self):
        return self.buf.shape[-1] if self.buf is not None else 0

    @property
    def ptr(self):
        return self.buf.data_ptr() + self.buf.element_size() * self.ch_off if self.buf is not None else None


class Conv:
    """one conv block's launch.  cin / ih / iw: its input; mat: the layer whose output it materialises (i + 1 when the
    epilogue absorbs the next block's shortcut or upsample); shortcut: that shortcut's source layer; s2d: a 3x3 / stride-2
    conv on an even grid with cin % 8 == 0, which the bf16 plans run as a 2x2-tap conv on a space-to-depth copy."""

    def __init__(self, model, i, shape, height, width):
        defs = model.module_defs
        d, seq = defs[i], model.module_list[i]
        nxt = defs[i + 1]["type"] if i + 1 < len(defs) else None
        self.i, self.k, self.stride = i, int(d["size"]), int(d["stride"])
        self.cout, self.oh, self.ow = shape[i]
        self.cin, self.ih, self.iw = (3, height, width) if i == 0 else shape[i - 1]
        # owner: the block whose weight a `weight_from` block borrows; such a block is a purely linear conv (no bias, BN
        # or activation, whatever its own modules hold).  dil: (dh, dw) of a [d-convolutional] block, else None.
        self.owner = int(d["weight_from"]) if "weight_from" in d else None
        self.dil = dilation(d) if d["type"] == "d-convolutional" else None
        if self.owner is not None:
            self.has_bn = self.has_act = False
        else:
            self.has_bn, self.has_act = hasattr(seq, "BatchNorm2d"), hasattr(seq, "activation")
        self.fuse_res = nxt == "shortcut" and i not in model.routes
        self.fuse_up = nxt == "upsample" and i not in model.routes and int(defs[i + 1]["stride"]) == 2
        # head = the linear, BN-less conv feeding a YOLO layer (or, in YOLO-less trunk graphs, any such conv)
        self.is_head = nxt == "yolo" or (not model.yolo_layers and not self.has_bn and not self.has_act)
        self.mat = i + 1 if (self.fuse_res or self.fuse_up) else i
        self.shortcut = None
        if self.fuse_res and not self.is_head:
            frm = int(defs[i + 1]["from"])
            self.shortcut = i + 1 + frm if frm < 0 else frm
        self.s2d = (self.stride == 2 and self.k == 3 and self.ih % 2 == 0 and self.iw % 2 == 0 and self.cin % 8 == 0)
        if self.dil is not None and (self.fuse_up or self.is_head):
            raise NotImplementedError("[d-convolutional] block %d feeding an upsample or a YOLO layer" % i)


class Graph:
    def __init__(self, model, height, width, accept, refuse):
        """accept: the block types beyond convolutional / route / shortcut / upsample / yolo that the plan runs ("se",
        "maxpool", "d-convolutional": the dilated convs and every `weight_from` block); any other type raises
        NotImplementedError(refuse % type)."""
        defs = self.defs = model.module_defs
        n = len(defs)
        shape = self.shape = [None] * n          # (C, H, W) of every block's output
        self.alias = {}                          # single-source route -> the layer whose output it is
        self.concats = {}                        # multi-source route -> its source layers
        c, h, w = 3, height, width
        for i, d in enumerate(defs):
            t = d["type"]
            if "weight_from" in d and "d-convolutional" not in accept:
                raise NotImplementedError(refuse % ("%s with weight_from" % t))
            if t == "convolutional" or (t == "d-convolutional" and t in accept):
                s = int(d["stride"])
                c, h, w = int(d["filters"]), (h + s - 1) // s, (w + s - 1) // s
            elif t == "upsample":
                h, w = h * int(d["stride"]), w * int(d["stride"])
            elif t == "maxpool" and t in accept:
                if int(d["size"]) != 2 or int(d["stride"]) not in (1, 2):
                    raise NotImplementedError("only the 2x2 max pools of yolov3-tiny have a kernel")
                if int(d["stride"]) == 2:
                    h, w = h // 2, w // 2
            elif t == "route":
                ls = route_sources(d, i)
                c = sum(shape[l][0] for l in ls)
                h, w = shape[ls[0]][1], shape[ls[0]][2]
                if len(ls) == 1:
                    self.alias[i] = self.alias.get(ls[0], ls[0])
                else:
                    if any(shape[l][0] % 8 for l in ls):
                        raise NotImplementedError("concat source with channels % 8 != 0")
                    self.concats[i] = ls
            elif t not in ("shortcut", "yolo") and t not in accept:
                raise NotImplementedError(refuse % t)
            shape[i] = (c, h, w)

        self.ops = []           # (block type, index) of every conv / se / maxpool launch, in execution order
        self.convs = {}         # conv index -> Conv
        made = set()            # layers whose output is materialised so far
        i = 0
        while i < n:
            t = defs[i]["type"]
            if t in ("convolutional", "d-convolutional"):
                cv = self.convs[i] = Conv(model, i, shape, height, width)
                if cv.shortcut is not None and (cv.shortcut not in made or shape[cv.shortcut] != shape[i]):
                    raise NotImplementedError("shortcut source layout")
                self.ops.append((t, i))
                if not cv.is_head:
                    made.add(cv.mat)
                i = cv.mat + 1
                continue
            if t in ("se", "maxpool"):
                self.ops.append((t, i))
                made.add(i)
            elif t == "route" and (i in self.concats or self.alias[i] in made):
                made.add(i)
            elif t in ("shortcut", "upsample"):
                raise NotImplementedError("%s at block %d does not follow a convolution it can be fused into" % (t, i))
            i += 1


class Buffers:
    """the output view of every materialised layer and, where the plan trains, its gradient twin.  alloc(h, w, cs)
    returns (buffer, gradient buffer or None) with channel stride cs; a layer outside any concat gets buffers of its own
    with cs rounded up to `round_to`.  channels: id of every buffer -> the channels its views cover (the rest of cs is
    padding no producer writes)."""

    def __init__(self, graph, alloc, round_to):
        self.graph, self.alloc, self.round_to = graph, alloc, round_to
        self.views, self.gviews = [None] * len(graph.shape), [None] * len(graph.shape)
        self.place = {}          # concat source -> (buffer, gradient buffer, channel offset)
        self.channels = {}
        for i, ls in graph.concats.items():
            c, h, w = graph.shape[i]
            buf, gbuf = alloc(h, w, L.round_up(c, 64))
            self._real(buf, gbuf, c)
            off = 0
            for l in ls:
                self.place[l] = (buf, gbuf, off)
                off += graph.shape[l][0]
            self.views[i], self.gviews[i] = self._pair(buf, gbuf, 0, c, h, w)

    def _real(self, buf, gbuf, c):
        for b in (buf, gbuf):
            if b is not None:
                self.channels[id(b)] = c

    @staticmethod
    def _pair(buf, gbuf, off, c, h, w):
        return View(buf, off, c, h, w), (View(gbuf, off, c, h, w) if gbuf is not None else None)

    def out(self, layer):
        """(view, gradient view or None) that `layer`'s producer writes: at its offset of its concat buffer, or fresh"""
        c, h, w = self.graph.shape[layer]
        if layer in self.place:
            buf, gbuf, off = self.place[layer]
        else:
            (buf, gbuf), off = self.alloc(h, w, L.round_up(c, self.round_to)), 0
            self._real(buf, gbuf, c)
        self.views[layer], self.gviews[layer] = self._pair(buf, gbuf, off, c, h, w)
        return self.views[layer], self.gviews[layer]

    def view(self, layer):
        return self.views[self.graph.alias.get(layer, layer)]

    def gview(self, layer):
        return self.gviews[self.graph.alias.get(layer, layer)]


def claim(written, view):
    """first-writer bookkeeping of the backward, walked last block first: True when earlier writes already cover the
    channel range of `view` (this write accumulates), False when it is the first (it overwrites).  written: buffer id ->
    the (lo, hi) channel ranges written so far."""
    key = id(view.buf)
    lo, hi = view.ch_off, view.ch_off + view.c
    covered = any(a <= lo and hi <= b for a, b in written.get(key, []))
    written.setdefault(key, []).append((lo, hi))
    return covered
