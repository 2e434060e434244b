"""One flat device buffer per Darknet model and mode (training bf16; eval bf16, one per batch size) that the
shape-sized storage of every plan comes from: the activations and their gradients, im2col / space-to-depth /
dilation-phase / zero-insert scratch, the SE scratch sized by the batch and the fp32 head buffers.  The reference's loops
change shape all the time (multi-scale training every 10 batches, the short last batch of every epoch, detect.py
--multi-scale on every image); with a pool the plan of each shape stays cached and holds only descriptors and small
tensors, and a switch allocates nothing.

Plans of different shapes overlay the same bytes, so at most one plan's data is live at a time:

  * ``build`` lays a plan out from offset 0.  The pool grows only when a shape needs more than it holds; growth first
    drops every plan laid out in the old storage (with their CUDA graphs), releases the old storage, allocates exactly
    the new requirement (zeroed) and lays the plan out again.  The old bytes return to the device only when nothing
    else holds a view of them: head tensors a caller still keeps from an earlier forward hold theirs.
  * ``activate`` runs before a plan's first launch whenever another plan used the storage since: the padded-NHWC
    buffers' zero halo and the channels no kernel writes are restored on the device (``ryolo_zero_halo_multi``).  The
    rest of each buffer is rewritten by every forward / step before it is read.
  * ``gen`` / ``consumed`` guard the fused training backward: it needs the activations of ITS forward, which the next
    forward of any shape overwrites."""
import torch

from . import _lib

ALIGN = 256           # every view starts at a multiple of this (TMA needs 16-byte addresses; the GEMMs' 128-byte rows)


class ActivationPool:
    def __init__(self, device):
        self.device = torch.device(device)
        self.storage = None           # uint8 [capacity]
        self.owner = None             # halo table of the plan whose zero invariants hold in the storage
        self.gen = 0                  # training forwards so far (the guard of the fused backward)
        self.consumed = True
        self._cursor = None
        self._jobs = None
        self._short = False

    @property
    def nbytes(self):
        return 0 if self.storage is None else self.storage.numel()

    def take(self, shape, dtype):
        """an uninitialised [shape] view of the storage (a stride-0 stand-in while the plan does not fit: build then
        grows the pool and lays the plan out again)"""
        if self._cursor is None:      # a plan built outside build() (a stand-alone TrainPlan): zeroed storage of its own
            return torch.zeros(shape, dtype=dtype, device=self.device)
        n = 1
        for s in shape:
            n *= int(s)
        n *= torch.empty((), dtype=dtype).element_size()
        off = -(-self._cursor // ALIGN) * ALIGN
        self._cursor = off + n
        if self._cursor > self.nbytes:
            self._short = True
            return torch.empty((1,) * len(shape), dtype=dtype, device=self.device).expand(*shape)
        return self.storage[off:off + n].view(dtype).view(shape)

    def padded(self, batch, h, w, cs, c_real):
        """[B, H+2, W+2, cs] bf16 whose halo, and channels [c_real, cs) of every pixel, are zero when the plan runs its
        first step (c_real = 0: the whole buffer; the kernels' write pattern decides, see the call sites; None: set by
        channels() before the plan's construction ends).  Outside build(): a zeroed tensor of its own."""
        t = self.take((batch, h + 2, w + 2, cs), torch.bfloat16)
        if self._jobs is not None:
            self._jobs.append([t, batch, h, w, c_real, cs])
        return t

    def channels(self, real):
        """c_real of the buffers padded() received as None: real = {id(buffer): channels} (graph.Buffers.channels)"""
        if self._jobs is not None:
            for j in self._jobs:
                if j[4] is None:
                    j[4] = real[id(j[0])]

    def build(self, make, drop):
        """plan = make() with its storage taken from this pool; returns (plan, halo table).  drop(): forget every plan
        laid out in the current storage (called before the storage is freed)."""
        plan, need, jobs = self._layout(make)
        if self._short:
            del plan, jobs
            drop()
            self.owner = None
            self.storage = None       # freed before the larger buffer is allocated
            # zeroed like the tensors of a plan built outside a pool: a grown pool holds no bytes of earlier work
            self.storage = torch.zeros(need, dtype=torch.uint8, device=self.device)
            plan, need2, jobs = self._layout(make)
            if self._short or need2 != need:
                raise RuntimeError("activation pool: the plan's layout changed between two passes (%d -> %d bytes)"
                                   % (need, need2))
        for t, b, h, w, c, cs in jobs:
            if c is None or not 0 <= c <= cs or cs % 8:
                raise ValueError("padded buffer [%d, %d, %d, %d]: real channels %s" % (b, h + 2, w + 2, cs, c))
        halo = [_lib.HaloJob(t.data_ptr(), b, h, w, c, cs, 0) for t, b, h, w, c, cs in jobs]
        arr = (_lib.HaloJob * len(halo))(*halo)
        table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self.device) if halo else None
        return plan, (table, len(halo))

    def _layout(self, make):
        self._cursor, self._jobs, self._short = 0, [], False
        try:
            plan = make()
            return plan, self._cursor, self._jobs
        finally:
            self._cursor, self._jobs = None, None

    def activate(self, halo, stream):
        """before the first launch of the plan whose halo table this is: restore its zero invariants when the storage
        served another plan (or none) since"""
        table, n = halo
        if self.owner is table:
            return
        if n:
            _lib.check(_lib.lib.ryolo_zero_halo_multi(_lib.ptr(table), n, stream), "ryolo_zero_halo_multi")
        self.owner = table

    def check(self, gen):
        """the backward of training forward `gen` needs that forward's activations: a later forward of any shape
        overwrote them, or a backward already turned z into dz in place.  Stock autograd would handle or reject these
        cases; silently wrong gradients are not an option."""
        if self.gen != gen or self.consumed:
            raise RuntimeError("Darknet training plan: the activations of this forward were overwritten by a later "
                               "forward (of any shape) or already consumed by a backward (retain_graph / two forwards "
                               "before one backward are not supported by the fused training path)")
