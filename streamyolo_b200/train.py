"""The training step around ``loss.backward()``: what the reference's trainer loop does per iteration
(/root/reference/exps/train_utils/double_trainer.py:99-123, 171-175), on flat fp32 state.

  * ``build_optimizer`` / ``ModelEMA``: [yolox 0.3.0] Exp.get_optimizer (SGD, momentum 0.9, nesterov, three parameter groups:
    BatchNorm weights and biases without decay, conv / linear weights with weight decay 5e-4) and ModelEMA(model, 0.9998) as
    plain PyTorch -- the drop-in path, used when the reference's own Trainer drives ``model(inps, targets)`` /
    ``loss.backward()`` (the training forward returns a loss with a grad_fn, model/backward.py) -- and the bit-level
    reference of the fused kernel.
  * ``Trainer``: the H100-native step.  Parameters, gradients, momentum and the EMA copy live in FLAT fp32 buffers laid out in
    the order in which the backward walk finishes the gradients; every ``nn.Parameter`` / BatchNorm buffer of the model is a
    view into them (state_dict, checkpoints and ``model.parameters()`` are unchanged).
      - the weight-gradient / BatchNorm-gradient kernels write straight into the flat gradient buffer (``FlatSink``);
      - the buffer is cut into ~25 MB buckets; the moment the walk has enqueued the last gradient of a bucket, its NCCL
        all-reduce is launched on the communication stream and overlaps the rest of the walk (what DistributedDataParallel's
        reducer does for the reference, double_trainer.py:171; ``broadcast_buffers=False``: BatchNorm statistics stay local);
      - ONE launch (``sy_sgd_nesterov_ema_step``) then does unscale (1 / (world x loss scale)) + weight decay + momentum +
        nesterov + parameter update + EMA over the whole state;
      - conv operands are re-packed from the fp32 masters by ``sy_pack_conv_weight`` launches (engine.WEIGHT_EPOCH).
  * the step as CUDA graph(s): ``Trainer.capture`` / ``replay`` at one input size; for multi-scale training
    (``Exp.random_resize`` every 10 iterations) ``multiscale_sizes`` lists the sizes, ``Trainer.capture_sizes`` captures
    one step per size into one graph memory pool, ``Trainer.replay_size`` runs one.  Every graph of a Trainer reads lr,
    weight decay, momentum, 1 / (world x loss scale) and the EMA decay from ONE device block; each replay refills it from
    one of two pinned host slots, and a slot is rewritten only after the copy that last read it has run, because the
    host runs ahead of the device.
  * checkpoints (double_trainer.py:221-226, 285-318, 353-371): ``Trainer.state_dict`` / ``load_state_dict`` (exact
    continuation), ``reference_checkpoint`` / ``load_reference_checkpoint`` (the reference's file and ``--resume``),
    ``optimizer_state_dict`` in torch.optim.SGD format, ``all_reduce_norm`` (BatchNorm statistics averaged over the ranks).
"""
import copy
import math

import torch
import torch.distributed as dist
from torch import nn

from . import dist as sydist
from . import ops
from .model import backward, engine


def build_optimizer(model, lr, momentum=0.9, weight_decay=5e-4):
    pg0, pg1, pg2 = [], [], []          # BN weights | weights with decay | biases
    for _, m in model.named_modules():
        if hasattr(m, "bias") and isinstance(m.bias, nn.Parameter):
            pg2.append(m.bias)
        if isinstance(m, nn.BatchNorm2d):
            pg0.append(m.weight)
        elif hasattr(m, "weight") and isinstance(m.weight, nn.Parameter):
            pg1.append(m.weight)
    opt = torch.optim.SGD(pg0, lr=lr, momentum=momentum, nesterov=True)
    opt.add_param_group({"params": pg1, "weight_decay": weight_decay})
    opt.add_param_group({"params": pg2})
    return opt


class ModelEMA:
    def __init__(self, model, decay=0.9998, updates=0):
        self.ema = copy.deepcopy(model).eval()
        self.updates = updates
        self.decay = lambda x: decay * (1 - math.exp(-x / 2000))
        for p in self.ema.parameters():
            p.requires_grad_(False)

    @torch.no_grad()
    def update(self, model):
        self.updates += 1
        d = self.decay(self.updates)
        msd = model.state_dict()
        for k, v in self.ema.state_dict().items():
            if v.dtype.is_floating_point:
                v.mul_(d).add_((1.0 - d) * msd[k].detach())


def train_step(model, optimizer, x, targets, ema=None, grad_scale=1.0):
    """The step with stock PyTorch pieces (torch.optim.SGD, Python EMA, post-hoc bucketed all-reduce): the semantics
    reference of ``Trainer.step``."""
    for p in model.parameters():
        p.grad = None
    losses = backward.forward_backward(model, x, targets, grad_scale=grad_scale)
    sydist.allreduce_grads(model.parameters())
    if grad_scale != 1.0:
        for p in model.parameters():
            if p.grad is not None:
                p.grad.div_(grad_scale)
    optimizer.step()
    engine.WEIGHT_EPOCH += 1
    if ema is not None:
        ema.update(model)
    return losses


def multiscale_sizes(input_size=(600, 960), random_size=(50, 70)):
    """The distinct input sizes (h, w) multi-scale training runs at: what ``Exp.random_resize`` can draw
    (StreamYOLO's cfgs/s_s50_onex_dfp_tal_flip.py:138-157: ``size = randint(*random_size)``,
    ``(16 * int(size * h / w), 16 * size)``, every 10 iterations) plus ``input_size`` (the last epoch), in drawing order."""
    size_factor = input_size[0] * 1.0 / input_size[1]
    out = []
    for size in range(random_size[0], random_size[1] + 1):
        hw = (16 * int(size * size_factor), int(16 * size))
        if hw not in out:
            out.append(hw)
    if tuple(input_size) not in out:
        out.append(tuple(input_size))
    return out


# ------------------------------------------------------------------------------------------------ flat state
def conv_groups_forward_order(model):
    """The BaseConv launch groups of one training forward in launch order (the recording forward: model/engine.py
    pafpn_frames, dfp_fuse and TALHead.run with a tape): a CSPLayer's conv1 | conv2 and the first cls | reg tower convs of
    a head level run as one GEMM, everything else alone."""
    net, head = model.backbone, model.head
    bb = net.backbone
    out = []

    def bc(m):
        out.append((m,))

    def csp(m):
        out.append((m.conv1, m.conv2))
        for blk in m.m:
            bc(blk.conv1)
            bc(blk.conv2)
        bc(m.conv3)

    bc(bb.stem.conv)
    bc(bb.dark2[0]); csp(bb.dark2[1])
    bc(bb.dark3[0]); csp(bb.dark3[1])
    bc(bb.dark4[0]); csp(bb.dark4[1])
    bc(bb.dark5[0]); bc(bb.dark5[1].conv1); bc(bb.dark5[1].conv2); csp(bb.dark5[2])
    bc(net.lateral_conv0); csp(net.C3_p4); bc(net.reduce_conv1); csp(net.C3_p3)
    bc(net.bu_conv2); csp(net.C3_n3); bc(net.bu_conv1); csp(net.C3_n4)
    bc(net.jian2); bc(net.jian1); bc(net.jian0)
    for k in range(len(head.stems)):
        bc(head.stems[k])
        out.append((head.cls_convs[k][0], head.reg_convs[k][0]))
        bc(head.cls_convs[k][1]); bc(head.reg_convs[k][1])
    return out


_ALIGN = 64     # floats: every segment of the flat buffers starts 256-byte aligned


class FlatState:
    """Flat fp32 buffers holding the model's parameters (walk order), their gradients, momentum, and the EMA copy; re-points
    the module's tensors into them."""

    def __init__(self, model, ema=True, copies=1):
        """``copies``: how many copies of the BatchNorm buffers the state holds, one per virtual rank (``Trainer``'s
        ``virtual_ranks``).  Copy k of a float buffer sits ``k * n_buf`` floats after copy 0, so the fused step's EMA
        covers every copy; ``num_batches_tracked`` gets one int64 copy per rank in ``int_bufs``.  The module's buffers
        are views of the copy ``select`` chose last, copy 0 outside a step."""
        dev = next(model.parameters()).device
        groups = list(reversed(conv_groups_forward_order(model)))        # the order the walk finishes them in
        head = model.head
        levels = list(reversed(range(len(head.stems))))
        seg_a, seg_b = [], []                                            # (tensor, slot) lists: no decay | decay
        for k in levels:                                                 # the head prediction convs finish first
            seg_b += [head.reg_preds[k].weight, head.obj_preds[k].weight, head.cls_preds[k].weight]
            seg_a += [head.reg_preds[k].bias, head.obj_preds[k].bias, head.cls_preds[k].bias]
        for g in groups:
            seg_b.append([m.conv.weight for m in g])                     # adjacent: one weight-gradient launch covers the group
            seg_a.append([m.bn.weight for m in g])
            seg_a.append([m.bn.bias for m in g])
        covered = set()
        self.offset = {}                                                 # id(tensor) -> (offset, numel)
        cur = 0

        def place(item):
            nonlocal cur
            cur = (cur + _ALIGN - 1) // _ALIGN * _ALIGN
            for t in (item if isinstance(item, list) else [item]):
                assert id(t) not in covered
                covered.add(id(t))
                self.offset[id(t)] = (cur, t.numel())
                cur += t.numel()

        for it in seg_a:
            place(it)
        cur = (cur + _ALIGN - 1) // _ALIGN * _ALIGN
        self.decay_begin = cur
        self.order_b = []                                                # parameters of the decayed class in walk order
        for it in seg_b:
            place(it)
            self.order_b += it if isinstance(it, list) else [it]
        cur = (cur + _ALIGN - 1) // _ALIGN * _ALIGN
        self.n_param = cur
        params = list(model.parameters())
        missing = [n for n, p in model.named_parameters() if id(p) not in covered]
        assert not missing, f"parameters outside the launch plan: {missing[:5]}"
        bufs = [b for b in model.buffers() if b.dtype.is_floating_point]
        for b in bufs:
            place(b)
        cur = (cur + _ALIGN - 1) // _ALIGN * _ALIGN
        self.copies, self.n_buf = copies, cur - self.n_param
        self.n_total = self.n_param + copies * self.n_buf
        self.state = torch.zeros(self.n_total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(self.n_param, dtype=torch.float32, device=dev)
        self.mom = torch.zeros(self.n_param, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for t in params + bufs:
                o, n = self.offset[id(t)]
                v = self.state[o:o + n].view(t.shape)
                v.copy_(t.detach().float())
                t.data = v                                              # the module tensor is now a view of the flat state
            for p in params:
                o, n = self.offset[id(p)]
                p.grad = self.grad[o:o + n].view(p.shape)
            for k in range(1, copies):
                self.buffer_copy(k).copy_(self.buffer_copy(0))
        self.bufs = bufs
        self.int_bufs, self.int_copies = [], None
        if copies > 1:
            self.int_bufs = [b for b in model.buffers() if not b.dtype.is_floating_point]
            self.int_copies = torch.stack([b.detach() for b in self.int_bufs]).repeat(copies, 1)
        self.selected = 0
        self.select(0)
        self.ema = self.state.clone() if ema else None
        self.params = params

    def buffer_copy(self, k, buf=None):
        """copy ``k`` of the float-buffer region of ``buf`` (default: ``state``), flat"""
        buf = self.state if buf is None else buf
        return buf[self.n_param + k * self.n_buf:self.n_param + (k + 1) * self.n_buf]

    def select(self, k):
        """point the module's BatchNorm buffers (running statistics, ``num_batches_tracked``) at copy ``k``: the kernels
        read the buffer addresses when a launch is issued or recorded"""
        self.selected = k
        if self.copies == 1:
            return
        for b in self.bufs:
            o, n = self.offset[id(b)]
            b.data = self.state[o + k * self.n_buf:o + k * self.n_buf + n].view(b.shape)
        for i, b in enumerate(self.int_bufs):
            b.data = self.int_copies[k, i]

    def gview(self, p):
        o, n = self.offset[id(p)]
        return self.grad[o:o + n]

    def views(self, model, buf):
        """``model.state_dict()`` with every entry that lives in the flat state taken from ``buf`` (a buffer laid out like
        ``state``, e.g. ``ema``) as a view; the rest (num_batches_tracked) are the module's own tensors."""
        base = self.state.data_ptr()
        index = {base + 4 * o: (o, n) for (o, n) in self.offset.values()}
        if self.copies > 1:                                              # the buffers of the selected copy
            shift = self.selected * self.n_buf
            index.update({base + 4 * (o + shift): (o + shift, n) for (o, n) in (self.offset[id(b)] for b in self.bufs)})
        out = {}
        for k, t in model.state_dict().items():
            hit = index.get(t.data_ptr()) if t.dtype == torch.float32 else None
            out[k] = buf[hit[0]:hit[0] + hit[1]].view(t.shape) if hit else t
        return out

    def ema_state_dict(self, model):
        """state_dict of the EMA model ([yolox] ModelEMA.ema.state_dict()): float entries from the flat EMA copy, the rest
        (num_batches_tracked) as in the live model."""
        return {k: t.clone() for k, t in self.views(model, self.ema).items()}


class FlatSink:
    """Gradient sink of the backward walk that writes into ``FlatState.grad`` and launches the all-reduce of a bucket as
    soon as all of its gradients have been enqueued."""

    def __init__(self, fs: FlatState, uses, bucket_bytes=25 << 20, overlap=True, world=None):
        self.fs, self.uses, self.overlap = fs, uses, overlap
        self.world = (dist.get_world_size() if dist.is_initialized() else 1) if world is None else world
        self.touched = set()
        # buckets over the decayed class in walk order; the small no-decay class is one last bucket
        self.buckets = []                   # [start, end, pending parameter count]
        self.bucket_of = {}
        start, size, members = fs.decay_begin, 0, []
        for p in fs.order_b:
            o, n = fs.offset[id(p)]
            if members and size + 4 * n > bucket_bytes:
                self._close(start, o, members)
                start, size, members = o, 0, []
            members.append(p)
            size += 4 * n
        self._close(start, fs.n_param, members)
        small = [p for p in fs.params if fs.offset[id(p)][0] < fs.decay_begin]
        self._close(0, fs.decay_begin, small)
        self.work = []
        self.launched = []
        self.on_bucket = None
        self.accumulate_all = False         # begin(accumulate=True): every kernel adds onto the flat gradient
        self.complete = True                # begin(complete=False): no bucket completes in this walk

    def _close(self, a, b, members):
        if not members:
            return
        idx = len(self.buckets)
        self.buckets.append([a, b, len(members)])
        for p in members:
            self.bucket_of[id(p)] = idx

    # ---- buffers for the kernels
    def _first(self, key):
        acc = self.accumulate_all or key in self.touched
        self.touched.add(key)
        return acc

    def conv_weight(self, mods, cin, kh, kw, stem=False):
        o, _ = self.fs.offset[id(mods[0].conv.weight)]
        n = sum(m.conv.weight.numel() for m in mods)
        t = self.fs.grad[o:o + n]
        shape = tuple(mods[0].conv.weight.shape) if stem else (sum(m.conv.out_channels for m in mods), cin, kh, kw)
        return t.view(shape), self._first(("w", id(mods[0])))

    def bn(self, mods):
        c = sum(m.conv.out_channels for m in mods)
        og, _ = self.fs.offset[id(mods[0].bn.weight)]
        ob, _ = self.fs.offset[id(mods[0].bn.bias)]
        return self.fs.grad[og:og + c], self.fs.grad[ob:ob + c], self._first(("bn", id(mods[0])))

    def head(self, head, k):
        ws = [self.fs.gview(p).view(p.shape[0], p.shape[1]) for p in (head.reg_preds[k].weight, head.obj_preds[k].weight,
                                                                      head.cls_preds[k].weight)]
        bs = [self.fs.gview(p) for p in (head.reg_preds[k].bias, head.obj_preds[k].bias, head.cls_preds[k].bias)]
        return ws, bs, self.accumulate_all

    # ---- completion tracking / communication
    def done(self, params):
        for p in params:
            key = id(p)
            left = self.pending.get(key)
            if left is None:
                continue
            left -= 1
            self.pending[key] = left
            if left == 0:
                b = self.buckets[self.bucket_of[key]]
                b[2] -= 1
                if b[2] == 0 and self.overlap:
                    self._launch(b)

    def begin(self, model, accumulate=False, complete=True):
        """per walk: how many launches contribute to each parameter (a module recorded twice, e.g. DFP jian, finishes on its
        last launch).  Virtual ranks: the walks after a step's first one ``accumulate`` into the gradient the earlier walks
        left, and only the step's last walk is ``complete``: its launches finish the gradients and launch the buckets."""
        self.touched.clear()
        self.accumulate_all, self.complete = accumulate, complete
        self.pending = {}
        self.work, self.launched = [], []
        if not complete:
            return
        for g in conv_groups_forward_order(model):
            n = self.uses.get(id(g[0]), 1)
            for m in g:
                for p in (m.conv.weight, m.bn.weight, m.bn.bias):
                    self.pending[id(p)] = n
        head = model.head
        for k in range(len(head.stems)):
            for p in (head.reg_preds[k].weight, head.obj_preds[k].weight, head.cls_preds[k].weight, head.reg_preds[k].bias,
                      head.obj_preds[k].bias, head.cls_preds[k].bias):
                self.pending[id(p)] = 1
        for i, b in enumerate(self.buckets):
            b[2] = sum(1 for k, v in self.bucket_of.items() if v == i)

    def _launch(self, b):
        self.launched.append((b[0], b[1]))
        if self.world > 1:
            if self.on_bucket is not None:
                self.on_bucket(b[0], b[1])          # graph capture: the trainer cuts the graph here and owns the collective
            else:
                self.work.append(dist.all_reduce(self.fs.grad[b[0]:b[1]], op=dist.ReduceOp.SUM, async_op=True))

    def finish(self):
        if not self.complete:
            return
        for b in self.buckets:
            if (b[0], b[1]) not in self.launched:
                self._launch(b)
        for w in self.work:
            w.wait()                        # the compute stream waits for the communication stream; no host sync


class Trainer:
    """H100-native training loop body for YOLOX(DFPPAFPN, TALHead): ``step(x, targets, lr)`` on frame pairs ``x``
    [B, 6, H, W] and (future, current) labels; for the still-image baseline YOLOX(DFPPAFPN, PIPEHead) also on still frames
    [B, 3, H, W] and one label tensor (one backbone pass, model/backward.py ``_record``)."""

    def __init__(self, model, lr=0.01, momentum=0.9, weight_decay=5e-4, ema_decay=0.9998, use_ema=True,
                 bucket_bytes=25 << 20, overlap=True, skip_nonfinite=False, virtual_ranks=1):
        """``skip_nonfinite``: what ``GradScaler.step`` does for the reference's ``--fp16`` (double_trainer.py:113-119).
        Every optimiser step first checks the all-reduced flat gradient for NaN / +-inf on the device (sy_nonfinite_flag;
        every rank sees the same sums, so every rank decides the same); a flagged step leaves the parameters and momentum
        as they are, while the EMA copy still moves towards them with that step's decay and ``updates`` still counts, as
        ModelEMA.update does after a skipped step.  ``skipped_steps()`` reads the device counter (a synchronisation).
        The check reads the gradient before the unscale: with a loss scale of 1 or more the unscaled gradient is finite
        exactly when it is.

        ``virtual_ranks`` = K: this process runs K ranks of a data-parallel run one after another, so that W processes
        train as W x K ranks would (the reference's ``-d 8`` on fewer GPUs).  Every input batch holds K x B samples;
        virtual rank k owns rows k*B .. (k+1)*B - 1 of the frames and of the labels.  Each virtual rank has its own
        BatchNorm running statistics, ``num_batches_tracked`` and EMA buffers (``broadcast_buffers=False``); a step runs
        K recording forwards and reverse walks on the K shards with rank k's buffers, the walks accumulating into one
        flat gradient (the buckets are all-reduced over the W processes during the last walk), and the fused step
        applies the mean over W x K.  ``step`` / ``replay`` return virtual rank 0's losses, ``rank_losses`` all K;
        outside a step the module's buffers are rank 0's."""
        assert model.training and model.head.use_l1
        engine.require_bf16_training(model)
        if int(virtual_ranks) != virtual_ranks or virtual_ranks < 1:
            raise ValueError(f"Trainer: virtual_ranks must be a positive integer, got {virtual_ranks!r}")
        self.virtual_ranks = int(virtual_ranks)
        self.model = model
        self.fs = FlatState(model, ema=use_ema, copies=self.virtual_ranks)
        self._rank_loss = None                             # the loss vector of every virtual rank in the last step
        self.skip_nonfinite = bool(skip_nonfinite)
        dev = self.fs.state.device
        self._found_inf = torch.zeros(1, dtype=torch.float32, device=dev) if self.skip_nonfinite else None
        self._skipped = torch.zeros(1, dtype=torch.int32, device=dev) if self.skip_nonfinite else None
        self.lr, self.momentum, self.weight_decay = lr, momentum, weight_decay
        self.ema_decay, self.updates = ema_decay, 0
        self.bucket_bytes, self.overlap = bucket_bytes, overlap
        self.sink = None
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self._hyper, self._hyper_slot = None, 0            # the captured graphs' hyper-parameter block (_capture)
        self._graph, self._sized = None, {}                # what capture / capture_sizes captured
        engine.WEIGHT_EPOCH += 1
        self._build_repack()
        self._repack()

    # ---- conv operands: every (parameter, layout) pair of the model re-packed by ONE launch after each update
    def _build_repack(self):
        dev = self.fs.state.device
        self.pack = ops.PackBatch(dev)
        self._packed_groups = []
        stem = self.model.backbone.backbone.stem.conv
        dt = ops.pack_conv_weight(stem.conv.weight[:1]).dtype     # bf16 (fp32 only under the CPU emulation with fp32 "storage")
        for g in conv_groups_forward_order(self.model):
            ws = [m.conv.weight for m in g]
            _, cin, kh, kw = ws[0].shape
            ot = sum(w.shape[0] for w in ws)
            if g[0] is stem:
                out = torch.empty((ot, kh, 64), dtype=dt, device=dev)
                self.pack.add(ws[0], out, 2)
                self._packed_groups.append((g, out, None))
                continue
            fwd = torch.empty((ot, kh * kw, cin), dtype=dt, device=dev)
            dg = torch.empty((cin, kh * kw, ot), dtype=dt, device=dev)
            o0 = 0
            for w in ws:
                self.pack.add(w, fwd[o0:o0 + w.shape[0]], 0)
                self.pack.add(w, dg, 1, out_pitch=ot, co_offset=o0)
                o0 += w.shape[0]
            self._packed_groups.append((g, fwd, dg))

    def _repack(self):
        """run the batched pack and hand the buffers to the engine's operand caches (keys of the current WEIGHT_EPOCH)"""
        self.pack.run()
        for g, fwd, dg in self._packed_groups:
            ws = [m.conv.weight for m in g]
            if dg is None:
                engine.packed_operand(g[0], "_pk", ws, ops.pack_stem_weight, value=fwd)
                continue
            engine.packed_operand(g[0], "_pk" if len(g) == 1 else "_pk2", ws, ops.pack_conv_weight, value=fwd)
            engine.packed_operand(g[0], "_pkd", ws, ops.pack_conv_weight_dgrad, value=dg)

    def forward_backward(self, x, targets, loss_scale=1.0):
        """The recording forward and reverse walk of every virtual rank on its shard; returns virtual rank 0's loss
        vector.  Each rank's tape (activations, gradient arena) is dropped before the next rank records, so a captured
        step's pool holds the activations of one rank."""
        shards = self._shards(x, targets)
        losses = []
        for k, (xk, tk) in enumerate(shards):
            self.fs.select(k)
            T, loss = backward._record(self.model, xk, tk)
            if self.sink is None:
                self.sink = FlatSink(self.fs, dict(T.uses), self.bucket_bytes, self.overlap, self.world)
            self.sink.uses = dict(T.uses)
            self.sink.begin(self.model, accumulate=k > 0, complete=k == len(shards) - 1)
            with torch.no_grad():
                backward._walk(T, self.model.head, loss_scale, self.sink)
            del T
            losses.append(loss)
        self.fs.select(0)
        self._rank_loss = losses
        return losses[0]

    def _shards(self, x, targets):
        """[(frames, labels)] of the virtual ranks: rows k*B .. (k+1)*B - 1 of ``x`` and of each label tensor"""
        K = self.virtual_ranks
        if K == 1:
            return [(x, targets)]
        n = x.shape[0]
        labels = [targets] if torch.is_tensor(targets) else list(targets)
        if n % K or any(t.shape[0] != n for t in labels):
            raise ValueError(f"Trainer: a batch of {n} samples (labels {[tuple(t.shape) for t in labels]}) cannot be cut "
                             f"into {K} virtual ranks of equal size")
        b = n // K
        cut = [[t[k * b:(k + 1) * b] for t in labels] for k in range(K)]
        return [(x[k * b:(k + 1) * b], cut[k][0] if torch.is_tensor(targets) else tuple(cut[k])) for k in range(K)]

    def rank_losses(self):
        """The loss dicts of every virtual rank in the last step or replay, in rank order (device tensors; a replay
        overwrites those of the graph it replays)."""
        return [backward._loss_dict(v) for v in self._rank_loss]

    def _hyper_values(self, lr, loss_scale):
        d = self.ema_decay * (1 - math.exp(-self.updates / 2000)) if self.fs.ema is not None else 0.0
        return [self.lr if lr is None else lr, self.momentum, self.weight_decay,
                1.0 / (self.world * self.virtual_ranks * loss_scale), d, 1.0 - d]

    def optimizer_step(self, lr=None, loss_scale=1.0, found_inf=None, hyper=None):
        if hyper is None:
            self.updates += 1
        h = self._hyper_values(lr, loss_scale)
        guard = {}
        if self.skip_nonfinite and found_inf is not None:
            raise ValueError("optimizer_step: found_inf is not taken by a Trainer built with skip_nonfinite=True (it "
                             "computes its own flag)")
        if self.skip_nonfinite:
            ops.nonfinite_flag(self.fs.grad, self._found_inf, self._skipped)
            guard = {"found_inf": self._found_inf, "found_inf_ema": True}
        elif found_inf is not None:
            guard = {"found_inf": found_inf}
        ops.sgd_nesterov_ema_step(self.fs.state, self.fs.grad, self.fs.mom, self.fs.ema, self.fs.n_param, self.fs.decay_begin,
                                  h[0], h[1], h[2], inv_scale=h[3], nesterov=True, ema_decay=h[4], hyper=hyper, **guard)
        engine.WEIGHT_EPOCH += 1            # the conv operands follow the new masters: one batched re-pack launch
        self._repack()

    def step(self, x, targets, lr=None, loss_scale=1.0):
        loss = self.forward_backward(x, targets, loss_scale)
        self.optimizer_step(lr, loss_scale)
        return backward._loss_dict(loss)

    # ---- the whole step as CUDA graph(s) (the eager step is bound by the host's launch rate: ~800-1300 launches)
    def capture(self, x, targets, loss_scale=1.0, prologue=None):
        """Capture forward + backward + weight re-pack + optimiser step on static input buffers (``x`` / ``targets`` become the
        graph's inputs: copy new data into them, then ``replay(lr)``).  One process: ONE graph.  Several ranks: the walk is cut
        into one graph segment per gradient bucket; between two segments the host enqueues that bucket's NCCL all-reduce on the
        communication stream, where it overlaps the following segments (the collectives themselves stay outside the
        captured graphs); a last segment holds the optimiser step.  ``prologue``: a callable captured at the front of the
        graph, e.g. ``data.pair_transform(..., out=(x, targets))`` so that the static inputs are the uint8 frames.

        Before capturing, the step runs once eagerly on the inputs as they stand: that warm-up is a real training step at
        ``self.lr`` (``updates`` goes up by one; parameters, BatchNorm statistics, momentum and the EMA copy advance), so
        the first ``replay`` is the second step.  Returns the number of graph segments."""
        self._graph = None                                 # a second call replaces the first: its graph goes first
        keyed = None if prologue is None else lambda *_: prologue()
        self._graph = self._capture({None: (x, targets)}, keyed, loss_scale, restore=False)[None]
        return len(self._graph[0])

    def replay(self, lr=None):
        return self._replay(self._graph, lr)

    def _capture(self, inputs, prologue, loss_scale, restore):
        """Capture one step per entry of ``inputs`` ({key: (x, targets)}; ``prologue(key, x, targets)`` at the front of
        each) into ONE graph memory pool, after one eager warm-up step per entry on a side stream (allocator, lazy module
        attributes).  ``restore``: the warm-up steps are undone, the training state (and the skipped-step counter) is as
        before the call.  Returns {key: (plan, loss vector, loss_scale, (x, targets))}, a plan being [(graph segment, bucket
        all-reduced after it, or None)].  The loss vectors stay referenced, so no later capture in the pool takes them over;
        so do the static inputs, which every replay writes (prologue) and reads: freed while the graph lives, their memory
        would go to other tensors that each replay then overwrites."""
        if self._hyper is None:          # ONE block per Trainer, never reallocated: every captured graph reads its address
            self._hyper = torch.zeros(8, dtype=torch.float32, device=self.fs.state.device)
            self._hyper_slots = [(torch.zeros(8, dtype=torch.float32).pin_memory(), torch.cuda.Event()) for _ in range(2)]
        snapshot = copy.deepcopy(self.state_dict()) if restore else None
        skipped = self._skipped.clone() if restore and self._skipped is not None else None
        self.updates += 1
        self._stage_hyper(None, loss_scale)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for key, (x, targets) in inputs.items():
                if prologue is not None:
                    prologue(key, x, targets)
                self.forward_backward(x, targets, loss_scale)
                self.optimizer_step(hyper=self._hyper)
            if restore:
                self.load_state_dict(snapshot)
                if skipped is not None:
                    self._skipped.copy_(skipped)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()                           # the warm-up's blocks: device memory for the graphs' pool
        pool = torch.cuda.graph_pool_handle()
        graphs = {}
        for key, (x, targets) in inputs.items():
            plan, cur = [], None

            def begin():
                nonlocal cur
                cur = torch.cuda.CUDAGraph()
                cur.capture_begin(pool=pool)

            def end(bucket=None):
                cur.capture_end()
                plan.append((cur, bucket))

            def cut(a, b):
                end((a, b))
                begin()

            self.sink.on_bucket = cut if self.world > 1 else None
            with torch.cuda.stream(side):
                begin()
                if prologue is not None:
                    prologue(key, x, targets)
                self.forward_backward(x, targets, loss_scale)
                if self.world > 1:                         # the optimiser step waits for the collectives: its own segment
                    end()
                    begin()
                self.optimizer_step(hyper=self._hyper)
                end()
            self.sink.on_bucket = None
            graphs[key] = (plan, self._rank_loss, loss_scale, (x, targets))
            torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        return graphs

    def _replay(self, graph, lr):
        plan, losses, loss_scale, _ = graph
        self.updates += 1
        self._stage_hyper(lr, loss_scale)
        self._replay_plan(plan)
        self._rank_loss = losses
        return backward._loss_dict(losses[0])

    def _stage_hyper(self, lr, loss_scale):
        """the hyper-parameter block of the captured graphs for the step ``updates``, through two pinned slots: a slot is
        written again only after the copy that read it last has run (the host runs ahead of the device)"""
        self._hyper_slot ^= 1
        host, copied = self._hyper_slots[self._hyper_slot]
        copied.synchronize()
        host[:6] = torch.tensor(self._hyper_values(lr, loss_scale))
        self._hyper.copy_(host, non_blocking=True)
        copied.record()

    def _replay_plan(self, plan):
        works = []
        for i, (g, bucket) in enumerate(plan):
            if i == len(plan) - 1:
                for w in works:
                    w.wait()
            g.replay()
            if bucket is not None:
                works.append(dist.all_reduce(self.fs.grad[bucket[0]:bucket[1]], op=dist.ReduceOp.SUM, async_op=True))

    # ---- multi-scale training: one captured step per input size, all in one graph memory pool
    def capture_sizes(self, sizes, make_inputs, prologue=None, loss_scale=1.0):
        """Capture one whole step (as ``capture``) per input size (``multiscale_sizes()``), for ``replay_size``.

        make_inputs(size) -> (x, targets)   the static input buffers of that size's graph; called for every size before
                                            anything is captured, so they live outside the graphs' memory pool;
                                            the sizes' inputs may be views of one buffer (one graph runs at a time);
                                            the Trainer keeps them referenced as long as their graphs
        prologue(size, x, targets)          captured at the front of that size's graph, fills its inputs: e.g.
                                            ``data.pair_transform(frames, ..., out=stage)`` into a buffer at ``input_size``
                                            followed by ``data.preprocess(*stage, size, input_size, out=(x, targets))``

        The capture leaves the training state as it found it: parameters, BatchNorm statistics (and
        ``num_batches_tracked``), momentum, the EMA copy and ``updates`` are restored after the eager warm-up step that
        each size runs before its capture.  The graphs share ONE memory pool (a step's intermediates are freed when its
        capture ends, so the next capture reuses them: the pool is about one step of the largest size); the loss vector of
        each graph stays referenced, so no capture takes it over.  Replays must therefore run one at a time, on the current
        stream, which ``replay_size`` does.  Several ranks: the graphs are cut at the same gradient buckets for every size
        (the flat gradient layout does not depend on the input size)."""
        sizes = sorted({tuple(int(v) for v in s) for s in sizes}, key=lambda s: -s[0] * s[1])   # largest first: the
        inputs = {s: make_inputs(s) for s in sizes}                                          # pool grows once
        self._sized = {}                                   # a second call replaces the first: its graphs go first
        self._sized = self._capture(inputs, prologue, loss_scale, restore=True)
        buckets = [[b for _, b in plan] for plan, _, _, _ in self._sized.values()]
        assert all(b == buckets[0] for b in buckets), "the gradient buckets differ between input sizes"
        return {s: len(plan) for s, (plan, _, _, _) in self._sized.items()}

    def replay_size(self, size, lr=None):
        """One captured step at ``size`` (a size given to ``capture_sizes``); returns its loss dict.  Several ranks: every rank
        must replay the same size, as the reference's ``Exp.random_resize`` ensures (rank 0 draws it and broadcasts it)."""
        size = tuple(int(v) for v in size)
        if size not in self._sized:
            raise KeyError(f"replay_size: no graph captured for {size} (captured: {sorted(self._sized)})")
        return self._replay(self._sized[size], lr)

    def ema_state_dict(self, rank=0):
        """the EMA model's state_dict as virtual rank ``rank`` holds it (its own EMA BatchNorm buffers)"""
        return self._at_rank(rank, lambda: self.fs.ema_state_dict(self.model))

    def model_state_dict(self, rank=0):
        """a copy of ``model.state_dict()`` as virtual rank ``rank`` holds it (its own BatchNorm buffers)"""
        return self._at_rank(rank, lambda: {k: t.clone() for k, t in self.model.state_dict().items()})

    def _at_rank(self, rank, fn):
        if not 0 <= rank < self.virtual_ranks:
            raise ValueError(f"virtual rank {rank} of {self.virtual_ranks}")
        self.fs.select(rank)
        try:
            return fn()
        finally:
            self.fs.select(0)

    def skipped_steps(self):
        """How many optimiser steps ``skip_nonfinite`` has skipped so far (reads the device counter: a synchronisation);
        0 without ``skip_nonfinite``."""
        return 0 if self._skipped is None else int(self._skipped.item())

    # ---- training state: save, resume, BatchNorm statistics over the ranks
    # Loading copies into the buffers the step reads (fs.state, fs.mom, fs.ema, the modules' integer buffers) and never
    # rebinds them: graphs captured by capture / capture_sizes keep reading those addresses, and the modules' tensors are
    # views into the flat state.
    def state_dict(self):
        """The whole training state, for an EXACT continuation with ``load_state_dict``:

            "model"         model.state_dict() (parameters, BatchNorm statistics, num_batches_tracked)
            "optimizer"     optimizer_state_dict(): momentum in torch.optim.SGD format
            "ema"           the EMA model's state_dict (as ema_state_dict()), None without EMA
            "updates"       optimiser steps so far (the EMA decay ramp)
            "lr", "momentum", "weight_decay"
                            the Trainer's hyper-parameters (``lr`` is the default of steps that are given none)

        As with ``nn.Module.state_dict`` the tensors are views of the live buffers: the weights, the momentum and the EMA
        copy each share one storage, so ``torch.save`` writes each of them once.  ``copy.deepcopy`` it for a snapshot in
        memory.  BatchNorm statistics are per rank, so with several ranks each rank saves its own.

        With ``virtual_ranks`` K > 1, "model" and "ema" hold virtual rank 0's buffers and one more entry holds every
        rank's:

            "virtual_ranks" [{"buffers": the model's buffer entries, "ema": the EMA model's, or None}] x K"""
        sd = {"model": self.model.state_dict(), "optimizer": self.optimizer_state_dict(),
              "ema": None if self.fs.ema is None else self.fs.views(self.model, self.fs.ema),
              "updates": self.updates, "lr": self.lr, "momentum": self.momentum, "weight_decay": self.weight_decay}
        if self.virtual_ranks > 1:
            sd["virtual_ranks"] = [self._at_rank(k, self._rank_buffers) for k in range(self.virtual_ranks)]
        return sd

    def _rank_buffers(self):
        """the selected virtual rank's buffer entries of the model and of the EMA model, as views"""
        names = [n for n, _ in self.model.named_buffers()]
        ema = None if self.fs.ema is None else self.fs.views(self.model, self.fs.ema)
        return {"buffers": {n: t.detach() for n, t in self.model.named_buffers()},
                "ema": None if ema is None else {n: ema[n].detach() for n in names}}

    def load_state_dict(self, sd):
        """Continue from a ``state_dict()`` of a Trainer of the same architecture and EMA setting: the next step computes
        bit for bit what the saving Trainer's next step would have."""
        if (sd["ema"] is None) != (self.fs.ema is None):
            raise ValueError(f"load_state_dict: the state was saved {'without' if sd['ema'] is None else 'with'} EMA, "
                             f"this Trainer runs {'with' if self.fs.ema is not None else 'without'} it")
        ranks = sd.get("virtual_ranks")
        if (1 if ranks is None else len(ranks)) != self.virtual_ranks:
            raise ValueError(f"load_state_dict: the state holds {1 if ranks is None else len(ranks)} virtual ranks, this "
                             f"Trainer runs {self.virtual_ranks}")
        self._check_entries(sd["model"], "model")
        if self.fs.ema is not None:
            self._check_entries(sd["ema"], "ema")
        self.load_optimizer_state_dict(sd["optimizer"])
        self._load_model(sd["model"])
        if self.fs.ema is not None:
            with torch.no_grad():
                for k, t in self.fs.views(self.model, self.fs.ema).items():
                    if t.dtype == torch.float32:
                        t.copy_(sd["ema"][k])
        if ranks is not None:
            for k in range(self.virtual_ranks):
                self._at_rank(k, lambda: self._load_rank_buffers(ranks[k]))
        self.updates = int(sd["updates"])
        self.lr, self.momentum, self.weight_decay = sd["lr"], sd["momentum"], sd["weight_decay"]
        self._state_changed()

    def optimizer_state_dict(self):
        """What ``build_optimizer(model, lr, momentum, weight_decay).state_dict()`` holds after the same updates (yolox's
        three groups, BN weights | decayed weights | biases, indices in group order), with each parameter's
        ``momentum_buffer`` a view of its slice of the flat momentum.  Before the first update there is no per-parameter
        state, as in torch."""
        opt = build_optimizer(self.model, self.lr, self.momentum, self.weight_decay)
        if self.updates > 0:
            for g in opt.param_groups:
                for p in g["params"]:
                    o, n = self.fs.offset[id(p)]
                    opt.state[p]["momentum_buffer"] = self.fs.mom[o:o + n].view(p.shape)
        return opt.state_dict()

    def load_optimizer_state_dict(self, sd):
        """Momentum and hyper-parameters from a torch.optim.SGD state_dict of ``build_optimizer``'s groups (the reference's
        ``ckpt["optimizer"]`` or ``optimizer_state_dict()``).  A parameter without ``momentum_buffer`` gets zeros, which
        is what torch's first step amounts to.  The fused step runs one lr and momentum, nesterov, and weight decay on the
        decayed group only: other hyper-parameters raise ``ValueError``."""
        opt = build_optimizer(self.model, self.lr, self.momentum, self.weight_decay)
        opt.load_state_dict(sd)                            # torch checks the group count and sizes
        g = opt.param_groups
        lr, momentum, wd = g[0]["lr"], g[0]["momentum"], g[1]["weight_decay"]
        if (any(x["lr"] != lr or x["momentum"] != momentum or not x["nesterov"] or x["dampening"] != 0
                or x.get("maximize", False) for x in g) or g[0]["weight_decay"] != 0 or g[2]["weight_decay"] != 0):
            raise ValueError("load_optimizer_state_dict: hyper-parameters the fused SGD-nesterov step cannot run: "
                             + str([{k: v for k, v in x.items() if k != "params"} for x in g]))
        bufs = [(p, opt.state.get(p, {}).get("momentum_buffer")) for x in g for p in x["params"]]
        bad = [(tuple(b.shape), tuple(p.shape)) for p, b in bufs if b is not None and b.shape != p.shape]
        if bad:
            raise ValueError(f"load_optimizer_state_dict: momentum_buffer shapes do not match the parameters: {bad[:3]}")
        with torch.no_grad():
            for p, b in bufs:
                o, n = self.fs.offset[id(p)]
                if b is None:
                    self.fs.mom[o:o + n].zero_()
                else:
                    self.fs.mom[o:o + n].copy_(b.reshape(-1))
        self.lr, self.momentum, self.weight_decay = lr, momentum, wd

    def reference_checkpoint(self, start_epoch, best_ap=0.0):
        """The dict the reference trainer's ``save_ckpt`` writes (exps/train_utils/double_trainer.py:353-371):
        ``{"start_epoch", "model", "optimizer", "best_ap"}`` with "model" the EMA weights when EMA is on, otherwise the live
        weights, and "optimizer" in torch.optim.SGD format.  ``torch.save`` it on rank 0 after ``all_reduce_norm()``.
        Resuming from it (``load_reference_checkpoint`` or the reference's ``--resume``) is lossy by the reference's own
        design; ``state_dict()`` is the exact path."""
        model = self.model.state_dict() if self.fs.ema is None else self.fs.views(self.model, self.fs.ema)
        return {"start_epoch": start_epoch, "model": model, "optimizer": self.optimizer_state_dict(), "best_ap": best_ap}

    def load_reference_checkpoint(self, ckpt, updates):
        """The reference's ``--resume`` (``resume_train``, double_trainer.py:285-318, and the ModelEMA built after it,
        :173-175) on a checkpoint its ``save_ckpt`` or ``reference_checkpoint`` wrote: ckpt["model"] becomes the live
        weights and BatchNorm buffers, the momentum and hyper-parameters come from ckpt["optimizer"], the EMA copy restarts
        from the loaded weights and ``updates`` is set to ``updates`` (the reference passes ``max_iter * start_epoch``).
        Lossy: when the file was saved with EMA the live weights are replaced by the EMA weights, as in the reference;
        ``load_state_dict`` is the exact path.  Returns ``(start_epoch, best_ap)``.

        Fine-tuning from a yolox checkpoint (``-c yolox_l.pth``: a shape-tolerant load of ckpt["model"] only) is done on
        the model before the Trainer is built."""
        self._check_entries(ckpt["model"], "ckpt['model']")
        self.load_optimizer_state_dict(ckpt["optimizer"])
        self._load_model(ckpt["model"])
        with torch.no_grad():                              # every reference rank loads the same file
            for k in range(1, self.virtual_ranks):
                self.fs.buffer_copy(k).copy_(self.fs.buffer_copy(0))
                self.fs.int_copies[k].copy_(self.fs.int_copies[0])
        if self.fs.ema is not None:
            self.fs.ema.copy_(self.fs.state)
        self.updates = int(updates)
        self._state_changed()
        return ckpt["start_epoch"], ckpt.get("best_ap", 0)

    def all_reduce_norm(self):
        """[yolox] ``all_reduce_norm(model)``, which the reference runs before every evaluation and ``last_epoch`` checkpoint
        (double_trainer.py:223-226): every BatchNorm state entry becomes its mean over the ranks.  The statistics are per
        rank during training (``broadcast_buffers=False``); they are the flat state's float-buffer region, so this is ONE
        all-reduce (SUM, then / world: yolox's ``op="mean"``).  BatchNorm weights and biases (parameters, updated with the
        mean gradient) and num_batches_tracked are equal on all ranks already.  Runs on the current stream and is not meant
        for a captured graph.  No-op in one process of one virtual rank.

        With ``virtual_ranks`` K the mean is over W x K ranks: the K copies are summed in rank order, the sum is
        all-reduced over the W processes and divided by W x K, and every copy receives the mean."""
        if self.world * self.virtual_ranks == 1:
            return
        stats = self.fs.buffer_copy(0)
        for k in range(1, self.virtual_ranks):
            stats.add_(self.fs.buffer_copy(k))
        if self.world > 1:
            dist.all_reduce(stats, op=dist.ReduceOp.SUM)
        stats.div_(self.world * self.virtual_ranks)
        for k in range(1, self.virtual_ranks):
            self.fs.buffer_copy(k).copy_(stats)
        self._state_changed()

    def _load_rank_buffers(self, entry):
        live = self._rank_buffers()
        with torch.no_grad():
            for which in ("buffers", "ema"):
                if live[which] is None:
                    continue
                for n, t in live[which].items():
                    t.copy_(entry[which][n])

    def _check_entries(self, sd, what):
        want = self.model.state_dict()
        missing = [k for k in want if k not in sd]
        extra = [k for k in sd if k not in want]
        shape = [k for k in want if k in sd and tuple(sd[k].shape) != tuple(want[k].shape)]
        if missing or extra or shape:
            raise ValueError(f"{what}: not a state of this model's architecture: {len(missing)} keys missing {missing[:3]}, "
                             f"{len(extra)} unexpected {extra[:3]}, {len(shape)} of another shape {shape[:3]}")

    def _load_model(self, sd):
        with torch.no_grad():
            for k, t in self.model.state_dict().items():       # views of the flat state, and the integer buffers
                t.copy_(sd[k])

    def _state_changed(self):
        """the flat state was written outside the fused step: new operand cache keys, conv operands re-packed in place"""
        engine.WEIGHT_EPOCH += 1
        self._repack()
