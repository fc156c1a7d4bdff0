"""Layer executor: walks the module tree with NHWC bf16 views and launches the CUDA ops.

Train mode (``model.training``): every BaseConv = wgmma conv writing the raw bf16 result + per-tile
statistic partials  ->  bn_finalize (batch statistics, running-stat update)  ->  bn_act_apply
(normalise + activation + optional residual, written straight into its consumer's concat slice).
The two frames of a pair are batched through the shared-weight backbone as 2B images with
*grouped* statistics (group 0 = current frames, group 1 = support frames), which reproduces the
reference's two sequential passes (/root/reference/exps/model/dfp_pafpn.py:120,145) exactly,
including the order of the two running-statistic updates.

Eval mode: BatchNorm is folded into a per-channel scale/shift applied in the conv epilogue
together with the activation and the residual (what yolox ``fuse_model`` + ``fuseforward`` achieve).  The activation is
each BaseConv's own (``act_code``: SiLU, ReLU or LeakyReLU(0.1), as its ``act`` name says).

The recording forward of a training step (model/backward.py) is this same walk with a tape in the ``Ctx``: nothing is
updated in place, every op keeps what its backward needs and is recorded on the tape.

Activation storage: bf16 everywhere by default.  An eval-mode ``Ctx`` may store every activation and pack every conv
operand in fp16 instead (``dtype=torch.float16``, what ``model.activation_dtype = torch.float16`` selects): 11 significant
bits instead of 8, the precision of the reference's half-precision inference.  The fp16 operands live in their own cache
slots ("_pkh", "_pk2h") next to the bf16 ones, so switching back and forth re-packs nothing and leaves the bf16 operands
(and train.Trainer's re-packed ones) alone.
"""
import torch

from .. import ops
from ..ops import View


WEIGHT_EPOCH = 0  # bumped by whoever updates parameters through raw pointers (train.Trainer's fused optimiser kernel does
                  # not touch torch's version counters): part of every packed-operand cache key
TRACE = None      # debugging: set to a dict to capture every BaseConv's stored output by module name
CONV_IMPL = "tc"  # conv of the plain forward: "tc" (wgmma kernel) or "simt" (CUDA-core cross-check); a tape always runs "tc"


def name_modules(model):
    for n, m in model.named_modules():
        m._sy_name = n


def _trace(m, y):
    if TRACE is not None:
        TRACE[getattr(m, "_sy_name", str(id(m)))] = y.torch().permute(0, 3, 1, 2).float().cpu()


ACTIVATION_DTYPES = (torch.bfloat16, torch.float16)


def check_activation_dtype(dtype):
    if dtype not in ACTIVATION_DTYPES:
        raise ValueError(f"activation_dtype must be torch.bfloat16 or torch.float16, not {dtype}")
    return dtype


def require_bf16_training(model):
    """training stores bf16 activations: refuse a model (or any of its modules) switched to fp16 storage"""
    if any(getattr(m, "activation_dtype", torch.bfloat16) != torch.bfloat16 for m in model.modules()):
        raise NotImplementedError("fp16 activation storage runs the eval / streaming forwards only (training stores bf16)")


class Ctx:
    """Per-forward execution context.  ``tape`` (a ``backward.Tape``): the recording forward of a training step -- every op
    keeps what its backward needs and is recorded on the tape; None: the plain forward.  ``stat_updates=2``: every train-mode
    conv of this context applies its (single-group) batch statistics to the running statistics twice -- one pass over a
    batch standing for the reference's two identical passes over it (a still frame duplicated into a pair).  ``dtype``: the
    activation storage, bf16 or (eval, tensor-core conv only) fp16."""

    def __init__(self, train, n, split, device, tape=None, stat_updates=1, dtype=torch.bfloat16):
        self.train = train
        self.n = n              # images in the batched tensor
        self.split = split      # first image of statistics group 1 (== n: single group)
        self.groups = 2 if split < n else 1
        self.device = device
        self.tape = tape
        self.stat_updates = stat_updates
        self.impl = "tc" if tape is not None else CONV_IMPL
        self.dtype = check_activation_dtype(dtype)
        self.f16 = dtype == torch.float16
        if self.f16 and (train or tape is not None):
            raise NotImplementedError("fp16 activation storage runs the eval / streaming forwards only (training stores bf16)")
        if self.f16 and self.impl != "tc":
            raise NotImplementedError(f"fp16 activation storage runs on the tensor-core conv only, not CONV_IMPL={self.impl!r}")

    def rec(self, **kw):
        if self.tape is not None:
            self.tape.rec(**kw)

    def empty(self, n, h, w, c) -> View:
        """a fresh activation buffer in the storage dtype (the dtype is passed only where it is not the default)"""
        if self.f16:
            return View.empty(n, h, w, c, self.device, torch.float16)
        return View.empty(n, h, w, c, self.device)

    def slot(self, name):
        """the packed-operand cache slot of this storage: fp16 operands are kept next to the bf16 ones, not over them"""
        return name + "h" if self.f16 else name

    def pack(self, fn):
        """the packing function ``fn`` (ops.pack_*) producing operands in the storage dtype"""
        if self.f16:
            return lambda *ws: fn(*ws, dtype=torch.float16)
        return fn


def packed_operand(m, slot, ws, pack, value=None):
    """The conv operand held in attribute ``slot`` of module ``m`` ("_pk": its own forward operand, "_pk2": the conv1 | conv2
    pair it leads, "_pkd": the data-gradient operand): ``pack(*ws)``, cached until one of the weights ``ws`` changes (torch
    version counter, storage, device) or WEIGHT_EPOCH moves.  ``value``: install that buffer as the operand of the current
    weights instead of packing (train.Trainer's batched re-pack)."""
    key = tuple((w._version, w.data_ptr(), w.device) for w in ws) + (WEIGHT_EPOCH,)
    if value is not None:
        setattr(m, slot, value)
        setattr(m, slot + "_key", key)
    elif getattr(m, slot + "_key", None) != key:
        setattr(m, slot, pack(*ws))
        setattr(m, slot + "_key", key)
    return getattr(m, slot)


def _folded(m):
    """Eval: scale = gamma / sqrt(running_var + eps), shift = beta - running_mean * scale (fp32)."""
    bn = m.bn
    key = (bn.weight._version, bn.bias._version, bn.running_mean._version, bn.running_var._version,
           getattr(m, "_stats_epoch", 0), bn.weight.data_ptr(), bn.eps, WEIGHT_EPOCH)
    if getattr(m, "_fold_key", None) != key:
        with torch.no_grad():
            scale = bn.weight.float() * torch.rsqrt(bn.running_var.float() + bn.eps)
            shift = bn.bias.float() - bn.running_mean.float() * scale
        m._fold = (scale.contiguous(), shift.contiguous())
        m._fold_key = key
    return m._fold


SYNC_SLOTS = 1024
_SYNC_POOLS = {}      # (device, stream) -> [int32 tensor of 2 * SYNC_SLOTS counters, next slot, scope depth]


def _sync_pool(device):
    key = (str(device), torch.cuda.current_stream().cuda_stream if torch.device(device).type == "cuda" else 0)
    st = _SYNC_POOLS.get(key)
    if st is None:
        st = [torch.zeros(2 * SYNC_SLOTS, dtype=torch.int32, device=device), 0, 0]
        _SYNC_POOLS[key] = st
    return st


class forward_scope:
    """Outermost scope of one forward (YOLOX / DFPPAFPN / TALHead / a stand-alone block / the recording forward): rewinds the
    grid-barrier counter pool of the current stream, so that the first train-mode conv of the forward zeroes it (ONE memset
    per forward, captured into the CUDA graph with it).  Every launch then takes its own counter slot: a launch that was
    aborted, or a module used by two forwards, can no longer leave a stale count for the next launch (the kernels also
    leave their slot at zero when they complete).  Launches on ONE stream only: two concurrent train-mode convs would each
    need every SM for their grid barrier (include/streamyolo_sm100.h)."""

    def __init__(self, device):
        self.device = device
        self.st = _sync_pool(device)

    def __enter__(self):
        if self.st[2] == 0:
            self.st[1] = 0
        self.st[2] += 1
        return self

    def __exit__(self, *a):
        self.st[2] -= 1
        return False


def _sync(m, device):
    """Two zeroed counters for one train-mode conv launch (grid barrier + exit ticket), from the stream's pool."""
    st = _sync_pool(device)
    if st[1] == 0:
        st[0].zero_()
    i = st[1]
    st[1] = (i + 1) % SYNC_SLOTS
    return st[0][2 * i:2 * i + 2]


def _bn_seg(m, c_begin=0):
    bn = m.bn
    return (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked, c_begin)


_CAPTURE_STREAMS = {}


def graph_capture_stream(device):
    """The side stream to capture CUDA graphs of the forward on (``torch.cuda.graph(g, stream=...)``), one per device.  The
    same stream on every call: the grid-barrier counter pool is kept per stream, so repeated captures share one pool."""
    key = str(device)
    if key not in _CAPTURE_STREAMS:
        _CAPTURE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _CAPTURE_STREAMS[key]


def capture_graph(fn, device, pool=None):
    """``fn`` as a CUDA graph: run once on a side stream (which packs the conv operands and folds BatchNorm outside the
    graph), synchronised, then captured on ``graph_capture_stream(device)``, in ``pool`` if given."""
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(device).wait_stream(side)
    torch.cuda.synchronize(device)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, pool=pool, stream=graph_capture_stream(device)):
        fn()
    return g


def act_code(m):
    """the kernels' SY_ACT_* code of a BaseConv's activation (its ``act`` name: "silu" / "relu" / "lrelu")"""
    return ops.ACT_CODES[m.act_name]


def conv_bn_act(ctx: Ctx, mods, x: View, wpk, k, s, y: View, res: View = None, act=None, y_goff1=0, res_goff1=0,
                impl=None, kind="normal"):
    """Train mode: conv -> batch statistics -> BatchNorm (running-stat update) -> act (+res) into ``y``.  ``act``: the
    SY_ACT_* code, by default that of ``mods`` (which share one activation).
    Tensor-core path = 2 launches: the conv writes the raw bf16 result, accumulates the statistics and
    (grid barrier + parallel reduce in its tail) publishes scale/shift; then the normalise pass.  ``mods``: one BaseConv, or two whose
    outputs are concatenated along channels (CSPLayer conv1 | conv2).  With a tape the conv also writes the batch mean /
    inverse std: the backward reads them and the raw output.  ``kind="stem"``: the Focus stem, whose
    input needs no gradient."""
    kh, kw = (k, k) if isinstance(k, int) else k
    ho = (x.h + 2 * ((kh - 1) // 2) - kh) // s + 1
    wo = (x.w + 2 * ((kw - 1) // 2) - kw) // s + 1
    cout = sum(m.conv.out_channels for m in mods)
    T = ctx.tape
    raw = View.empty(x.n, ho, wo, cout, ctx.device)
    bn0 = mods[0].bn
    mom = float(0.1 if bn0.momentum is None else bn0.momentum)
    n = x.n
    split = ctx.split if ctx.groups == 2 else 0
    for m in mods:
        m._stats_epoch = getattr(m, "_stats_epoch", 0) + 1
    impl = impl or ctx.impl
    if act is None:
        act = act_code(mods[0])
    if impl == "tc":
        partials = torch.empty((ops.conv_stat_rows(), 4 * cout), dtype=torch.float32, device=ctx.device)
        segs, c0 = [], 0
        for m in mods:
            segs.append(_bn_seg(m, c0))
            c0 += m.conv.out_channels
        ss = torch.empty((2, 2, cout), dtype=torch.float32, device=ctx.device)
        mi = None if T is None else torch.empty((2, 2, cout), dtype=torch.float32, device=ctx.device)
        # the keyword only where it is not the default: every other launch is issued exactly as before it existed
        repeat = {} if ctx.stat_updates == 1 else {"stat_updates": ctx.stat_updates}
        ops.conv2d(x, wpk, raw, k, s, ops.SY_CONV_RAW, impl="tc", partials=partials, split_n=split, bn=segs,
                   momentum=mom, eps=float(bn0.eps), scale_shift=ss, sync=_sync(mods[0], ctx.device), mean_invstd=mi,
                   **repeat)
        ops.bn_act_apply(raw, ss[0].data_ptr(), ss[1].data_ptr(), split if split else n, act, res, y, y_goff1, res_goff1)
        if T is not None:
            T.rec(t="conv", mods=mods, x=x, k=(kh, kw), s=s, raw=raw, y=y, res=res, ss=ss, mi=mi, split=split, act=act,
                  kind=kind)
            T.uses[id(mods[0])] = T.uses.get(id(mods[0]), 0) + 1
        return
    # CUDA-core path (cross-check of the tensor-core kernel; depthwise convs): conv, separate statistics pass, separate
    # finalize per module, apply
    if ctx.stat_updates != 1:
        raise NotImplementedError(f"repeated running-statistics updates run on the tensor-core conv only, not impl={impl!r}")
    ops.conv2d(x, wpk, raw, k, s, ops.SY_CONV_RAW, impl=impl)
    sc = torch.empty((2, 2, cout), dtype=torch.float32, device=ctx.device)
    sp = split if split else n
    c0 = 0
    for m in mods:
        c = m.conv.out_channels
        P = ops.stats_num_partials(n, ho * wo)
        partials = torch.empty((P, 2, c), dtype=torch.float32, device=ctx.device)
        ops.channel_stats(raw.ch(c0, c), partials)
        tmp = torch.empty((2, 2, c), dtype=torch.float32, device=ctx.device)
        bn = m.bn
        ops.bn_finalize(partials, (P // n) * sp if split else 0, 2 if split else 1, sp * ho * wo,
                        bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked,
                        mom, float(bn.eps), tmp[0], tmp[1])
        sc[:, :, c0:c0 + c] = tmp
        c0 += c
    if y_goff1 == 0 and res_goff1 == 0:
        ops.bn_act_apply(raw, sc[0], sc[1], sp, act, res, y)
    else:   # group-1 images go to a shifted destination (DFP fusion): one call per group
        nb = sp
        ops.bn_act_apply(raw.imgs(0, nb), sc[0, 0], sc[1, 0], nb, act,
                         res.imgs(0, nb) if res is not None else None, y.imgs(0, nb))
        y1 = View(y.buf, y.c0, y.c, y.n0, nb).shifted(y_goff1 + nb * y.img_elems())
        r1 = View(res.buf, res.c0, res.c, res.n0, nb).shifted(res_goff1 + nb * res.img_elems()) if res is not None else None
        ops.bn_act_apply(raw.imgs(nb, nb), sc[0, 1], sc[1, 1], nb, act, r1, y1)


def base_conv(ctx: Ctx, m, x: View, y: View = None, res: View = None) -> View:
    """[yolox] BaseConv: act(bn(conv(x))) (+ res).  ``y`` may be a slice of a concat buffer.  Also takes a [yolox] DWConv
    (depthwise BaseConv then pointwise BaseConv) wherever the reference's ``Conv = DWConv if depthwise else BaseConv`` puts one."""
    if hasattr(m, "dconv"):
        return base_conv(ctx, m.pconv, base_conv(ctx, m.dconv, x), y, res)
    k, s = m.ksize, m.stride
    ho, wo = ops.conv_out_hw(x.h, x.w, k, s)
    cout = m.conv.out_channels
    if y is None:
        y = ctx.empty(x.n, ho, wo, cout)
    dw = m.conv.groups > 1
    wpk = packed_operand(m, ctx.slot("_pk"), [m.conv.weight], ctx.pack(ops.pack_dw_weight if dw else ops.pack_conv_weight))
    impl = "dw" if dw else ctx.impl
    act = act_code(m)
    if not ctx.train:
        scale, shift = _folded(m)
        ops.conv2d(x, wpk, y, k, s, ops.SY_CONV_FUSED, impl=impl, scale=scale, shift=shift, act=act, res=res)
    else:
        conv_bn_act(ctx, (m,), x, wpk, k, s, y, res, act, impl=impl)
    _trace(m, y)
    return y


def _folded_pair(m1, m2):
    a, b = _folded(m1), _folded(m2)
    key = (id(a[0]), id(b[0]))
    if getattr(m1, "_fold2_key", None) != key:
        m1._fold2 = (torch.cat([a[0], b[0]]).contiguous(), torch.cat([a[1], b[1]]).contiguous())
        m1._fold2_key = key
    return m1._fold2


def conv_pair(ctx: Ctx, m1, m2, x: View) -> View:
    """Two BaseConvs with the same geometry reading the same input as ONE launch: [.., c1 + c2] output, one BatchNorm
    parameter segment per module (CSPLayer conv1 | conv2; the first cls / reg tower convs of a head level).  Depthwise
    variants, and two modules with different activations, take two ordinary launches into the one buffer."""
    if hasattr(m1, "dconv") or hasattr(m2, "dconv") or m1.act_name != m2.act_name:
        c1, c2 = (getattr(m, "pconv", m).conv.out_channels for m in (m1, m2))
        u = ctx.empty(x.n, x.h, x.w, c1 + c2)
        base_conv(ctx, m1, x, u.ch(0, c1))
        base_conv(ctx, m2, x, u.ch(c1, c2))
        return u
    c1, c2 = m1.conv.out_channels, m2.conv.out_channels
    k, s = m1.ksize, m1.stride
    assert (m2.ksize, m2.stride, m2.conv.in_channels) == (k, s, m1.conv.in_channels)
    ho, wo = ops.conv_out_hw(x.h, x.w, k, s)
    u = ctx.empty(x.n, ho, wo, c1 + c2)
    wpk = packed_operand(m1, ctx.slot("_pk2"), [m1.conv.weight, m2.conv.weight], ctx.pack(ops.pack_conv_weight))
    if not ctx.train:
        scale, shift = _folded_pair(m1, m2)
        ops.conv2d(x, wpk, u, k, s, ops.SY_CONV_FUSED, impl=ctx.impl, scale=scale, shift=shift, act=act_code(m1))
    else:
        conv_bn_act(ctx, (m1, m2), x, wpk, k, s, u)
    _trace(m1, u.ch(0, c1))
    _trace(m2, u.ch(c1, c2))
    return u


def csp_layer(ctx: Ctx, m, x: View, out: View = None) -> View:
    """[yolox] CSPLayer: conv3(cat(m(conv1 x), conv2 x)).  conv1 and conv2 read the same input, so they
    run as ONE GEMM with 2*hidden output channels written straight into the concat buffer; the
    bottleneck chain then updates the first half in place.  No concat copy ever happens -- except with a tape: the
    backward needs every input kept, so the chain runs in fresh buffers, its last output lands in a second concat buffer
    and conv2's half is copied next to it."""
    hid = m.conv1.conv.out_channels
    u = conv_pair(ctx, m.conv1, m.conv2, x)
    a = u.ch(0, hid)
    keep = ctx.tape is not None
    if keep:
        u2 = View.empty(x.n, x.h, x.w, 2 * hid, ctx.device)
    for i, blk in enumerate(m.m):
        t = base_conv(ctx, blk.conv1, a)
        dst = a
        if keep:
            dst = u2.ch(0, hid) if i == len(m.m) - 1 else View.empty(x.n, x.h, x.w, hid, ctx.device)
        base_conv(ctx, blk.conv2, t, dst, res=a if blk.use_add else None)
        a = dst
    if keep:
        if len(m.m) == 0:
            copy(ctx, a, u2.ch(0, hid))
        copy(ctx, u.ch(hid, hid), u2.ch(hid, hid))
        u = u2
    return base_conv(ctx, m.conv3, u, out)


def copy(ctx: Ctx, src: View, dst: View):
    ops.copy(src, dst)
    ctx.rec(t="copy", src=src, dst=dst)


def focus_stem(ctx: Ctx, m, x, frames) -> View:
    """[yolox] Focus + BaseConv straight from the NCHW float frame-pair batch: space-to-depth + W-gather into
    a 64-channel NHWC tensor, then the tensor-core kernel runs the 3x3 stem as a 3x1 conv (3 K blocks)."""
    b, ch, h, w = x.shape
    bc = m.conv
    cout = bc.conv.out_channels
    n = frames * b
    xin = ctx.empty(n, h // 2, w // 2, 64)
    ops.focus_pack(x, frames, xin)
    wpk = packed_operand(bc, ctx.slot("_pk"), [bc.conv.weight], ctx.pack(ops.pack_stem_weight))
    y = ctx.empty(n, h // 2, w // 2, cout)
    if not ctx.train:
        scale, shift = _folded(bc)
        ops.conv2d(xin, wpk, y, ops.STEM_K, 1, ops.SY_CONV_FUSED, impl=ctx.impl, scale=scale, shift=shift,
                   act=act_code(bc))
    else:
        conv_bn_act(ctx, (bc,), xin, wpk, ops.STEM_K, 1, y, kind="stem")
    _trace(bc, y)
    return y


def spp_bottleneck(ctx: Ctx, m, x: View) -> View:
    hid = m.conv1.conv.out_channels
    s = ctx.empty(x.n, x.h, x.w, 4 * hid)
    base_conv(ctx, m.conv1, x, s.ch(0, hid))
    ops.spp_maxpool(s.ch(0, hid), s.ch(hid, hid), s.ch(2 * hid, hid), s.ch(3 * hid, hid))
    ctx.rec(t="spp", x=s.ch(0, hid), y5=s.ch(hid, hid), y9=s.ch(2 * hid, hid), y13=s.ch(3 * hid, hid))
    return base_conv(ctx, m.conv2, s)


def upsample(ctx: Ctx, x: View, y: View):
    ops.upsample_nearest(x, y)
    ctx.rec(t="upsample", x=x, y=y)


def darknet(ctx: Ctx, bb, x, frames, dark3: View = None, dark4: View = None):
    """CSPDarknet stem -> dark5 for ``frames`` x B images (/root/reference/exps/model/darknet.py:167-179).  ``dark3`` /
    ``dark4``: where the dark3 / dark4 outputs go (e.g. slices of the PAFPN's concat buffers).  Returns the (stem, dark2,
    dark3, dark4, dark5) views."""
    outs = [focus_stem(ctx, bb.stem, x, frames)]
    for blk, dst in ((bb.dark2, None), (bb.dark3, dark3), (bb.dark4, dark4)):
        outs.append(csp_layer(ctx, blk[1], base_conv(ctx, blk[0], outs[-1]), dst))
    t = base_conv(ctx, bb.dark5[0], outs[-1])
    t = spp_bottleneck(ctx, bb.dark5[1], t)
    outs.append(csp_layer(ctx, bb.dark5[2], t))
    return outs


def pafpn_frames(ctx: Ctx, net, x, frames):
    """CSPDarknet + PAFPN for ``frames`` x B images (/root/reference/exps/model/darknet.py:167-179,
    dfp_pafpn.py:120-140).  Returns the un-fused (pan_out2, pan_out1, pan_out0) views."""
    c3 = net.C3_p3.conv3.conv.out_channels
    c4 = net.C3_p4.conv3.conv.out_channels
    n = frames * x.shape[0]
    h8, w8 = x.shape[2] // 2, x.shape[3] // 2                       # Focus, then the 3x3 stride-2 convs of dark2, dark3
    for _ in range(2):
        h8, w8 = ops.conv_out_hw(h8, w8, 3, 2)
    h16, w16 = ops.conv_out_hw(h8, w8, 3, 2)
    f1 = ctx.empty(n, h8, w8, 2 * c3)                    # cat(up(fpn_out1), dark3)
    f0 = ctx.empty(n, h16, w16, 2 * c4)                  # cat(up(fpn_out0), dark4)
    x0 = darknet(ctx, net.backbone, x, frames, f1.ch(c3, c3), f0.ch(c4, c4))[-1]
    h32, w32 = x0.h, x0.w
    z0 = ctx.empty(n, h32, w32, 2 * c4)                  # cat(bu_conv1, fpn_out0)
    fpn0 = base_conv(ctx, net.lateral_conv0, x0, z0.ch(c4, c4))
    upsample(ctx, fpn0, f0.ch(0, c4))
    fo0 = csp_layer(ctx, net.C3_p4, f0)
    z1 = ctx.empty(n, h16, w16, 2 * c3)                  # cat(bu_conv2, fpn_out1)
    fpn1 = base_conv(ctx, net.reduce_conv1, fo0, z1.ch(c3, c3))
    upsample(ctx, fpn1, f1.ch(0, c3))
    pan2 = csp_layer(ctx, net.C3_p3, f1)
    base_conv(ctx, net.bu_conv2, pan2, z1.ch(0, c3))
    pan1 = csp_layer(ctx, net.C3_n3, z1)
    base_conv(ctx, net.bu_conv1, pan1, z0.ch(0, c4))
    pan0 = csp_layer(ctx, net.C3_n4, z0)
    return pan2, pan1, pan0


def dfp_fuse(ctx: Ctx, net, cur, sup):
    """Dual-Flow Perception fusion (/root/reference/exps/model/dfp_pafpn.py:168-170, 211-221):
    out = cat(jian(cur), jian(sup)) + cur, a single bf16 rounding after the residual add.
    ``cur`` / ``sup`` are per-level views with the same image count."""
    outs = []
    for m, c, s in zip((net.jian2, net.jian1, net.jian0), cur, sup):
        nb = c.n
        if hasattr(m, "dconv"):                               # depthwise=True: jian is a DWConv (dfp_pafpn.py:83-105)
            half = m.pconv.conv.out_channels
            out = ctx.empty(nb, c.h, c.w, 2 * half)
            sub = Ctx(ctx.train, nb, nb, ctx.device, ctx.tape, dtype=ctx.dtype)   # two calls = two BatchNorm batches, like the reference
            base_conv(sub, m, c, out.ch(0, half), res=c.ch(0, half))
            base_conv(sub, m, s, out.ch(half, half), res=c.ch(half, half))
            outs.append(out)
            continue
        half = m.conv.out_channels
        out = ctx.empty(nb, c.h, c.w, 2 * half)
        wpk = packed_operand(m, ctx.slot("_pk"), [m.conv.weight], ctx.pack(ops.pack_conv_weight))
        act = act_code(m)
        if not ctx.train:
            scale, shift = _folded(m)
            ops.conv2d(c, wpk, out.ch(0, half), 1, 1, ops.SY_CONV_FUSED, impl=ctx.impl, scale=scale, shift=shift,
                       act=act, res=c.ch(0, half))
            ops.conv2d(s, wpk, out.ch(half, half), 1, 1, ops.SY_CONV_FUSED, impl=ctx.impl, scale=scale,
                       shift=shift, act=act, res=c.ch(half, half))
        else:
            # the reference runs jian(cur) then jian(sup): two BN batches, two running-stat updates.
            # Batched here (grouped statistics) when cur/sup are the two halves of one buffer -- not with a tape: the
            # backward takes one statistics group per launch.
            same = (c.buf is s.buf) and s.n0 == c.n0 + nb and c.c0 == s.c0 and c.c == s.c
            if same and ctx.tape is None:
                both = View(c.buf, c.c0, c.c, c.n0, 2 * nb)
                sub = Ctx(True, 2 * nb, nb, ctx.device)
                # group 1 (support frames, images nb..2nb-1) lands in channels [half, 2*half) of image n - nb
                yv = View(out.buf, 0, half, 0, 2 * nb)
                rv = View(c.buf, c.c0, half, c.n0, 2 * nb)
                conv_bn_act(sub, (m,), both, wpk, 1, 1, yv, rv, act,
                            y_goff1=half - nb * yv.img_elems(), res_goff1=half - nb * rv.img_elems())
            else:
                sub = Ctx(True, nb, nb, ctx.device, ctx.tape)
                for src, dst, r in ((c, out.ch(0, half), c.ch(0, half)), (s, out.ch(half, half), c.ch(half, half))):
                    conv_bn_act(sub, (m,), src, wpk, 1, 1, dst, r, act)
        outs.append(out)
    return tuple(outs)


def as_view(t, dtype=torch.bfloat16) -> View:
    """Accept a View or an NCHW-shaped torch tensor (zero-copy when it is channels-last ``dtype``, bf16 or fp16)."""
    if isinstance(t, View):
        return t
    p = t.permute(0, 2, 3, 1)
    if t.dtype == dtype and p.is_contiguous():
        return View(p)
    return View(p.contiguous().to(dtype))


def as_nchw(v: View):
    """NCHW-shaped (channels-last memory) tensor over a view, as the reference API returns."""
    return v.torch().permute(0, 3, 1, 2)
