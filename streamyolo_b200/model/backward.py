"""Training step with gradients: a recording forward + the reverse walk over the recorded kernels.

    losses = backward.forward_backward(model, x, (labels_future, labels_current))     # fills p.grad of every parameter

What ``loss.backward()`` does for the reference (/root/reference/exps/train_utils/double_trainer.py:110-114) through
exps/model/{yolox,dfp_pafpn,darknet,tal_head}.py, expressed over the kernels of libstreamyolo_sm100 (DESIGN.md 4.3):

  * the forward is the engine's walk of the product's forward (model/engine.py: same kernels, same batching of the two
    frames with grouped BatchNorm statistics) run with a ``Tape``, which makes the two differences a backward pass needs:
    nothing is updated in place (every conv keeps its input, its raw output and the batch statistics), and the DFP fusion
    runs its two jian convs as two launches;
  * every recorded op then runs its backward in reverse order.  Gradients of activations live in bf16 buffers that mirror
    the activation buffers (a channel / image slice of an activation is the same slice of its gradient buffer) and are
    *accumulated*: a tensor read by several consumers (Bottleneck shortcuts, FPN features, the concat buffers) simply
    receives several contributions -- the conv data gradient accumulates through the FUSED epilogue's residual input.
  * parameter gradients are fp32 in PyTorch's layouts (conv OIHW, BN weight / bias, pred-conv weight / bias) and are added
    to ``p.grad`` like autograd does.

Where the parameter gradients go is decided by a *gradient sink*: ``TensorSink`` (fresh fp32 tensors, what autograd /
``forward_backward`` hand out) or ``train.FlatSink`` (slices of the trainer's flat gradient buffer in walk order, whose
buckets are all-reduced over NCCL as soon as their last gradient has been enqueued -- the overlap DistributedDataParallel
gives the reference, /root/reference/exps/train_utils/double_trainer.py:171).

Every kernel used here is tested on the GPU against autograd, the routing on CPU with the kernels emulated in torch
(tests/test_cpu_backward.py), the assembled walk on the GPU against autograd through the oracle
(tests/test_gpu_model.py::test_forward_backward_vs_oracle_autograd, tests/test_gpu_train.py).  ``YOLOX.forward`` in training
mode with gradients enabled returns ``loss_with_autograd`` (the step as one autograd node)."""
import torch

from . import engine
from .pipe_head import PIPEHead
from .tal_head import _f32
from .. import ops
from ..ops import View


DEBUG_HOOK = None     # tests: callable(stage, record, **tensors) invoked inside the walk (tests/test_gpu_train.py checks every
                      # recorded conv's backward in situ against torch on the very tensors the kernels saw)


POISON = False        # tests: fill the gradient arena with NaN instead of leaving it uninitialised -- a region that is read
                      # before anything was written to it then poisons the parameter gradients (tests/test_cpu_backward.py)


class Tape:
    def __init__(self, device):
        self.device = device
        self.ops = []
        self.gbuf = {}          # id(activation buffer) -> gradient buffer (bf16)
        self.keep = []          # keeps the activation buffers (and so their ids) alive
        self.uses = {}          # id(BaseConv) -> number of recorded launches (a module used twice accumulates: DFP jian)
        self.cover = {}         # id(activation buffer) -> bool [images, channels]: which part of its gradient has been written
        self.pending = {}       # id(activation buffer) -> [(dst view, src gradient view)]: deferred first contributions (see defer)

    def g(self, v: View) -> View:
        key = id(v.buf)
        if key not in self.gbuf:
            self.gbuf[key] = torch.zeros_like(v.buf)                 # (not in the arena: zero-filled, i.e. written)
            self.cover[key] = torch.ones((v.buf.shape[0], v.buf.shape[3]), dtype=torch.bool)
            self.keep.append(v.buf)
        return View(self.gbuf[key], v.c0, v.c, v.n0, v.n)

    # The arena is NOT zero-filled (the memset plus the reads of those zeros by every first accumulation were ~0.9 ms of a
    # 20 ms StreamYOLO-l step).  Instead the walk asks before every gradient write whether the region already holds a
    # contribution: the first contribution is WRITTEN (copy instead of add, the conv data gradient without its residual
    # input), later ones accumulate; a region that is read before any consumer wrote to it is zero-filled on the spot
    # (a tensor without consumers -- does not happen in this network, kept for safety).  Host-side bookkeeping only.
    def _cov(self, v: View):
        c = self.cover[id(v.buf)]
        return c[v.n0:v.n0 + v.n, v.c0:v.c0 + v.c]

    def _zero_uncovered(self, v: View):
        """zero-fill the not yet written part of the gradient region of ``v`` (rectangles of equal image rows)"""
        cov = self._cov(v)
        gb = self.gbuf[id(v.buf)]
        n = 0
        while n < v.n:
            m = n + 1
            while m < v.n and torch.equal(cov[m], cov[n]):
                m += 1
            row = cov[n]
            c = 0
            while c < v.c:
                if row[c]:
                    c += 1
                    continue
                e = c
                while e < v.c and not row[e]:
                    e += 1
                gb[v.n0 + n:v.n0 + m, :, :, v.c0 + c:v.c0 + e].zero_()
                c = e
            n = m
        cov[:] = True

    # A shortcut's gradient (g(res) += g(y)) that would be the FIRST contribution to g(res) is not copied: it is remembered and
    # handed to the conv data-gradient launch that writes the same region next, as that launch's residual input
    # (g(x) = conv(...) + g(y) in one epilogue).  Any other access to the region first materialises the copy.
    @staticmethod
    def _same(a: View, b: View):
        return a.buf is b.buf and (a.c0, a.c, a.n0, a.n) == (b.c0, b.c, b.n0, b.n)

    @staticmethod
    def _overlap(a: View, b: View):
        return (a.buf is b.buf and a.c0 < b.c0 + b.c and b.c0 < a.c0 + a.c and a.n0 < b.n0 + b.n and b.n0 < a.n0 + a.n)

    def defer(self, src: View, v: View):
        """g(v) (+)= src, deferred when it would be the first write"""
        self.g(v)
        self._resolve(v)
        if bool(self._cov(v).any()):
            self.accumulate(src, v)
        else:
            self.pending.setdefault(id(v.buf), []).append((v, src))

    def take_pending(self, v: View):
        """the deferred source for EXACTLY the region of ``v`` (removed from the table), or None; other deferred regions that
        overlap ``v`` are materialised"""
        lst = self.pending.get(id(v.buf), [])
        hit = None
        for i, (dv, src) in enumerate(lst):
            if self._same(dv, v):
                hit = lst.pop(i)[1]
                break
        self._resolve(v)
        return hit

    def _resolve(self, v: View):
        lst = self.pending.get(id(v.buf))
        if not lst:
            return
        keep = []
        for dv, src in lst:
            if self._overlap(dv, v):
                gd = View(self.gbuf[id(dv.buf)], dv.c0, dv.c, dv.n0, dv.n)
                cov = self._cov(dv)
                if not bool(cov.any()):
                    cov[:] = True
                    ops.copy(src, gd)
                else:
                    if not bool(cov.all()):
                        self._zero_uncovered(dv)
                    ops.add_(src, gd)
            else:
                keep.append((dv, src))
        self.pending[id(v.buf)] = keep

    def first(self, v: View) -> bool:
        """True: nothing has been written to the gradient of ``v`` yet -- the caller must WRITE it (the region counts as
        written from now on); False: it holds contributions -- the caller accumulates."""
        self._resolve(v)
        cov = self._cov(v)
        if not bool(cov.any()):
            cov[:] = True
            return True
        if not bool(cov.all()):
            self._zero_uncovered(v)              # partly written: complete it with zeros, then accumulate
        return False

    def gread(self, v: View) -> View:
        """gradient of ``v`` for READING: everything that was never written is zero"""
        g = self.g(v)
        self._resolve(v)
        if not bool(self._cov(v).all()):
            self._zero_uncovered(v)
        return g

    def accumulate(self, src: View, v: View):
        """g(v) (+)= src"""
        g = self.g(v)
        if self.first(v):
            ops.copy(src, g)
        else:
            ops.add_(src, g)

    def prepare_grads(self):
        """ONE uninitialised arena holding the gradient buffer of every activation buffer the walk will touch, instead of
        one allocation per buffer (see ``first`` for why it needs no memset)."""
        bufs, seen = [], set()

        def add(v):
            if v is not None and id(v.buf) not in seen and id(v.buf) not in self.gbuf:
                seen.add(id(v.buf))
                bufs.append(v.buf)

        for r in self.ops:
            t = r["t"]
            if t == "conv":
                add(r["y"]); add(r["res"])
                if r["kind"] != "stem":
                    add(r["x"])
            elif t == "copy":
                add(r["dst"]); add(r["src"])
            elif t == "upsample":
                add(r["y"]); add(r["x"])
            elif t == "spp":
                for k in ("x", "y5", "y9", "y13"):
                    add(r[k])
            elif t == "head":
                for _, cf, rf, _ in r["levels"]:
                    add(cf); add(rf)
        if not bufs:
            return
        sizes = [(b.numel() + 127) // 128 * 128 for b in bufs]            # 256-byte aligned slots
        arena = torch.empty(sum(sizes), dtype=bufs[0].dtype, device=self.device)
        if POISON:
            arena.fill_(float("nan"))
        off = 0
        for b, n in zip(bufs, sizes):
            self.gbuf[id(b)] = arena[off:off + b.numel()].view(b.shape)
            self.cover[id(b)] = torch.zeros((b.shape[0], b.shape[3]), dtype=torch.bool)
            self.keep.append(b)
            off += n

    def rec(self, **kw):
        self.ops.append(kw)


class TensorSink:
    """Gradient sink that hands out fresh fp32 tensors (one per launch group, the members' gradients are views of it)."""

    def __init__(self, device):
        self.device = device
        self.store = {}         # key -> tensor
        self.seen = set()
        self.views = {}         # id(parameter) -> gradient view

    def _get(self, key, shape, params, splits):
        """tensor for ``key`` (+ whether it already holds a contribution); ``params`` / ``splits``: the parameters it covers
        along dim 0"""
        if key in self.store:
            return self.store[key], True
        t = torch.empty(shape, dtype=torch.float32, device=self.device)
        self.store[key] = t
        o = 0
        for p, n in zip(params, splits):
            self.views[id(p)] = t[o:o + n].view(p.shape) if tuple(t[o:o + n].shape) != tuple(p.shape) else t[o:o + n]
            o += n
        return t, False

    def conv_weight(self, mods, cin, kh, kw, stem=False):
        couts = [m.conv.out_channels for m in mods]
        if stem:                # the stem's gradient arrives in the packed layout and is unpacked by the caller
            return self._get(("ws", id(mods[0])), tuple(mods[0].conv.weight.shape), [mods[0].conv.weight], [couts[0]])
        return self._get(("w", id(mods[0])), (sum(couts), cin, kh, kw), [m.conv.weight for m in mods], couts)

    def bn(self, mods):
        couts = [m.conv.out_channels for m in mods]
        g, acc = self._get(("g", id(mods[0])), (sum(couts),), [m.bn.weight for m in mods], couts)
        b, _ = self._get(("b", id(mods[0])), (sum(couts),), [m.bn.bias for m in mods], couts)
        return g, b, acc

    def head(self, head, k):
        ps = (head.reg_preds[k].weight, head.obj_preds[k].weight, head.cls_preds[k].weight,
              head.reg_preds[k].bias, head.obj_preds[k].bias, head.cls_preds[k].bias)
        out = []
        for p in ps:
            shape = (p.shape[0], p.shape[1]) if p.dim() == 4 else tuple(p.shape)
            t, _ = self._get(("h", id(p)), shape, [p], [p.shape[0]])
            out.append(t)
        return out[:3], out[3:], False

    def done(self, params):
        pass

    def finish(self):
        pass

    def grad_of(self, p):
        return self.views.get(id(p))


# ------------------------------------------------------------------------------------------------ reverse walk
def _conv_backward(T: Tape, r, sink):
    mods, x, raw, y, res = r["mods"], r["x"], r["raw"], r["y"], r["res"]
    kh, kw = r["k"]
    s = r["s"]
    dev = T.device
    cout, cin = raw.c, x.c
    stem = r["kind"] == "stem"
    gy = T.gread(y)
    if res is not None:
        T.defer(gy, res)                                         # shortcut / "+ cur" branch
    draw = View.empty(raw.n, raw.h, raw.w, cout, dev)
    dgamma, dbeta, acc_bn = sink.bn(mods)
    if DEBUG_HOOK is not None:
        DEBUG_HOOK("pre", r, gy=gy, dgamma=dgamma, dbeta=dbeta, acc_bn=acc_bn)
    ops.bn_act_backward(raw, gy, draw, r["ss"][0], r["ss"][1], r["mi"][0], r["mi"][1], r["split"], r["act"], dgamma, dbeta,
                        accumulate=acc_bn)
    if stem:
        # packed stem weights: wpk[o][row r][s * 16 + fc] = w[o][fc][r][s]  ->  dw[o][s * 16 + fc][r][0]
        dw = torch.empty((cout, cin, kh, kw), dtype=torch.float32, device=dev)
        ops.conv2d_wgrad(x, draw, (kh, kw), s, dw)
        gw, acc_w = sink.conv_weight(mods, cin, kh, kw, stem=True)
        g = dw[:, :48, :, 0].reshape(cout, 3, 16, 3)[:, :, :12, :].permute(0, 2, 3, 1)     # [o, s, fc, r] -> [o, fc, r, s]
        if acc_w:
            gw.add_(g)
        else:
            gw.copy_(g)
        sink.done([mods[0].conv.weight, mods[0].bn.weight, mods[0].bn.bias])
        return                                                    # the input frames need no gradient
    dw, acc_w = sink.conv_weight(mods, cin, kh, kw)
    gx = T.g(x)
    shortcut = T.take_pending(x)                                  # a deferred shortcut gradient for exactly this region
    fresh = T.first(x)                                            # no consumer has written this input's gradient yet
    assert shortcut is None or fresh
    if DEBUG_HOOK is not None:
        DEBUG_HOOK("pre_w", r, dw=dw, acc_w=acc_w, gx=shortcut if shortcut is not None else (None if fresh else gx))
    ops.conv2d_wgrad(x, draw, (kh, kw), s, dw, accumulate=acc_w)
    sink.done([p for m in mods for p in (m.conv.weight, m.bn.weight, m.bn.bias)])
    one, zero = _one_zero(T, cin)
    src = draw
    if s == 2:
        src = View.empty(x.n, x.h, x.w, cout, dev)
        ops.dilate2(draw, src)
    # data gradient: gx = conv(src, flipped / transposed filter) * 1 + 0 (+ gx: accumulated in place through the residual input)
    wpk = engine.packed_operand(mods[0], "_pkd", [m.conv.weight for m in mods], ops.pack_conv_weight_dgrad)
    ops.conv2d(src, wpk, gx, (kh, kw), 1, ops.SY_CONV_FUSED, scale=one, shift=zero, act=0,
               res=shortcut if shortcut is not None else (None if fresh else gx))
    if DEBUG_HOOK is not None:
        DEBUG_HOOK("post", r, draw=draw, dgamma=dgamma, dbeta=dbeta, dw=dw, gx=gx)


def _one_zero(T, c):
    """per-channel scale 1 / shift 0 of the data-gradient launches (one pair of constants per width and tape)"""
    cache = T.__dict__.setdefault("_oz", {})
    if c not in cache:
        cache[c] = (torch.ones(c, dtype=torch.float32, device=T.device), torch.zeros(c, dtype=torch.float32, device=T.device))
    return cache[c]


NARROW_HEAD_CLASSES = 27     # sy_head_pred_backward's register accumulators; above it sy_head_pred_backward_wide


def _head_backward(T: Tape, head, r, grad_scale, sink):
    out, origin = r["out"], r["origin"]
    g_raw = torch.empty_like(out)
    ops.tal_loss_backward(out, origin, r["fut"], r["hw"], head.strides, float(head.gamma), True, r["ws"], grad_scale,
                          grad_raw=g_raw)
    pred_backward = ops.head_pred_backward if head.num_classes <= NARROW_HEAD_CLASSES else ops.head_pred_backward_wide
    for k, cf, rf, off in r["levels"]:
        regp, objp, clsp = head.reg_preds[k], head.obj_preds[k], head.cls_preds[k]
        dws, dbs, acc = sink.head(head, k)
        gcf, grf = T.g(cf), T.g(rf)
        assert T.first(cf) and T.first(rf), "the prediction convs are the only consumers of the tower outputs"
        pred_backward(g_raw, cf, rf, gcf, grf, _f32(regp.weight), _f32(objp.weight), _f32(clsp.weight),
                      r["a_total"], off, dws[0], dws[1], dws[2], dbs[0], dbs[1], dbs[2], accumulate=acc)
        sink.done([regp.weight, objp.weight, clsp.weight, regp.bias, objp.bias, clsp.bias])


def _walk(T: Tape, head, grad_scale, sink):
    T.prepare_grads()
    for r in reversed(T.ops):
        t = r["t"]
        if t == "conv":
            _conv_backward(T, r, sink)
        elif t == "head":
            _head_backward(T, head, r, grad_scale, sink)
        elif t == "copy":
            T.accumulate(T.gread(r["dst"]), r["src"])
        elif t == "upsample":
            x = r["x"]
            gy, gx = T.gread(r["y"]), T.g(x)
            if T.first(x):
                ops.upsample_nearest_backward(gy, gx)
            else:
                tmp = View.empty(x.n, x.h, x.w, x.c, T.device)
                ops.upsample_nearest_backward(gy, tmp)
                ops.add_(tmp, gx)
        elif t == "spp":
            x = r["x"]
            g5, g9, g13, gx = T.gread(r["y5"]), T.gread(r["y9"]), T.gread(r["y13"]), T.g(x)
            if T.first(x):
                ops.spp_maxpool_backward(x, g5, g9, g13, gx)
            else:
                tmp = View.empty(x.n, x.h, x.w, x.c, T.device)
                ops.spp_maxpool_backward(x, g5, g9, g13, tmp)
                ops.add_(tmp, gx)
        else:
            raise RuntimeError(t)
    assert not any(T.pending.values()), "deferred shortcut gradients left over"
    sink.finish()


def label_pair(model, targets):
    """(future, current) labels of a training batch.  A ``PIPEHead`` (the still-image baseline,
    /root/reference/exps/model/pipe_head.py) takes ONE label tensor and uses it for both, as ``PIPEHead.forward`` does; the
    TAL head needs the pair (indexing a single tensor would take the labels of images 0 and 1)."""
    if not torch.is_tensor(targets):
        return targets
    if not isinstance(model.head, PIPEHead):
        raise TypeError(f"{type(model.head).__name__} trains on (future labels, current labels); got one label tensor "
                        f"{tuple(targets.shape)} (only PIPEHead takes a single tensor)")
    return targets, targets


def _record(model, x, targets):
    """Recording forward of YOLOX(DFPPAFPN, TALHead / PIPEHead) in train mode; returns (tape, loss vector [total, iou, conf,
    cls, l1, num_fg]).

    ``x`` [B, 6, H, W]: frame pairs, the two frames batched as 2B images with grouped statistics.  ``x`` [B, 3, H, W]: still
    frames.  The reference duplicates them into identical pairs (dfp_pafpn.py:236-238), so its second backbone + PAFPN pass
    repeats the first: same activations, same batch statistics, a second running-statistics update, and a backward that
    is linear in the incoming gradient.  Here ONE pass runs over the B frames with each BatchNorm's running update applied
    twice (stat_updates=2), and the DFP fusion reads that pass as both cur and sup, so the gradients of the two branches
    meet in the same buffer."""
    assert model.training and model.head.use_l1
    if any(getattr(m, "groups", 1) > 1 for m in model.modules() if isinstance(m, torch.nn.Conv2d)):
        raise NotImplementedError("the training backward does not cover depthwise convolutions (depthwise=True): forward only")
    engine.require_bf16_training(model)
    targets = label_pair(model, targets)
    net = model.backbone
    xin = x.float().contiguous()
    b = xin.shape[0]
    if xin.shape[1] not in (3, 6):
        raise ValueError(f"training input must be [B, 6, H, W] frame pairs or [B, 3, H, W] still frames, got {tuple(xin.shape)}")
    dev = xin.device
    T = Tape(dev)
    with torch.no_grad(), engine.forward_scope(dev):
        if xin.shape[1] == 3:
            pans = engine.pafpn_frames(engine.Ctx(True, b, b, dev, T, stat_updates=2), net, xin, 1)
            cur = sup = pans
        else:
            pans = engine.pafpn_frames(engine.Ctx(True, 2 * b, b, dev, T), net, xin, 2)
            cur = tuple(p.imgs(0, b) for p in pans)
            sup = tuple(p.imgs(b, b) for p in pans)
        ctx = engine.Ctx(True, b, b, dev, T)
        fused = engine.dfp_fuse(ctx, net, cur, sup)       # jian: two launches, one running update each (as the reference)
        loss = model.head.run(ctx, fused, targets)
    return T, loss


def _loss_dict(loss):
    return {"total_loss": loss[0], "iou_loss": loss[1], "l1_loss": loss[4], "conf_loss": loss[2], "cls_loss": loss[3],
            "num_fg": loss[5]}


def forward_backward(model, x, targets, grad_scale=1.0, sink=None):
    """One training forward + backward of YOLOX(DFPPAFPN, TALHead) in train mode on a frame-pair batch ``x`` [B, 6, H, W]
    (or of a still model, YOLOX(DFPPAFPN, PIPEHead), on ``x`` [B, 3, H, W] and one label tensor; see ``_record``).
    Returns the loss dict of YOLOX.forward (0-dim tensors).  Without ``sink`` the gradients are accumulated into ``p.grad``
    of every parameter (like autograd); with a sink (train.FlatSink) they are written where the sink says."""
    T, loss = _record(model, x, targets)
    own = sink is None
    if own:
        sink = TensorSink(T.device)
    with torch.no_grad():
        _walk(T, model.head, grad_scale, sink)
    if own:
        for p in model.parameters():
            g = sink.grad_of(p)
            if g is not None:
                g = g.to(p.dtype)
                p.grad = g if p.grad is None else p.grad + g
    return _loss_dict(loss)


class _TrainLoss(torch.autograd.Function):
    """The whole training forward as ONE autograd node: forward = recording forward, backward = the reverse walk.  The
    parameters are inputs of the node, so ``loss.backward()`` hands their gradients to autograd like any other op --
    optimizers, ``GradScaler`` (the incoming gradient is the loss scale) and ``DistributedDataParallel``'s reducer hooks see
    nothing unusual (/root/reference/exps/train_utils/double_trainer.py:105-123, 171)."""

    @staticmethod
    def forward(ctx, model, x, fut, cur, *params):
        T, loss = _record(model, x, (fut, cur))
        ctx.tape, ctx.model, ctx.params = T, model, params
        ctx.mark_non_differentiable(loss)
        return loss[0].clone(), loss

    @staticmethod
    def backward(ctx, g_total, _g_all):
        T, model = ctx.tape, ctx.model
        sink = TensorSink(T.device)
        with torch.no_grad():
            _walk(T, model.head, float(g_total), sink)    # one host sync per step: the loss scale as a kernel argument
        grads = tuple(None if sink.grad_of(p) is None else sink.grad_of(p).to(p.dtype) for p in ctx.params)
        ctx.tape = None
        return (None, None, None, None) + grads


def loss_with_autograd(model, x, targets):
    """Loss dict whose ``total_loss`` carries a grad_fn (see _TrainLoss); the other entries are detached values."""
    params = tuple(p for p in model.parameters() if p.requires_grad)
    fut, cur = label_pair(model, targets)
    total, loss = _TrainLoss.apply(model, x, fut, cur, *params)
    d = _loss_dict(loss)
    d["total_loss"] = total
    return d
