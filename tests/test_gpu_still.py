"""GPU: training the still-image baseline, YOLOX(DFPPAFPN, PIPEHead) on single frames (cfgs/l_s50_still_dfp_flip.py), with
one backbone + PAFPN pass per frame instead of the reference's two identical ones (model/backward.py ``_record``).

  * sy_conv2d_tc with stat_updates = 2: the running statistics are the kernel's own batch mean / variance applied twice
    (fp64 reference), num_batches_tracked += 2, and everything else the launch writes is bit-identical to stat_updates = 1
  * the single pass against the duplicated pair on the same StreamYOLO-s model at 600 x 960: losses, parameter gradients and
    running statistics
  * every recorded conv's backward checked in situ on the still model (the walk takes paths the pair network never takes)
  * the reference trainer's call sequence (GradScaler) and Trainer.capture / replay on 3-channel batches
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import DFPPAFPN, PIPEHead, YOLOX, backward  # noqa: E402
from streamyolo_b200.ops import View  # noqa: E402
from test_gpu_model import ORDER  # noqa: E402
from test_gpu_ops import rand_w  # noqa: E402

DEV = "cuda"


def build_still(depth, width, momentum=0.03):
    ch = [256, 512, 1024]
    m = YOLOX(DFPPAFPN(depth, width, in_channels=ch), PIPEHead(8, width, in_channels=ch))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, momentum
    m.head.initialize_biases(1e-2)
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}), strict=True)
    m.head.use_l1 = True
    return m.cuda().train()


def still_batch(b, h, w, seed=4321):
    x = synth.synth_frames(b, h, w, seed=seed)[:, :3].contiguous().cuda()
    labels, _ = synth.synth_labels(b, h, w, seed=11)
    return x, labels.cuda()


# ------------------------------------------------------------------------------------------------ 1. the kernel
# shapes of tests/test_gpu_parity_l.py (StreamYOLO-l, 8 pairs): a 1x1 conv on linear tiles and a 3x3 stride-1 conv on halo tiles
@pytest.mark.parametrize("tile_bn", [64, 128])
@pytest.mark.parametrize("case", [(8, 256, 256, 75, 120, 1, 1), (8, 256, 256, 75, 120, 3, 1)], ids=["linear", "halo"])
def test_conv_stat_updates_twice(case, tile_bn):
    n, ci, co, h, w, k, s = case
    tile_mode = 2 if k == 3 else 1
    plan = ops.conv2d_plan(n, h, w, ci, co, k, s, tile_mode=tile_mode, tile_bn=tile_bn)
    assert (plan["mode"], plan["bn"]) == (tile_mode, tile_bn)
    g = torch.Generator(device=DEV).manual_seed(1)
    xb = torch.randn((n, h, w, ci), generator=g, device=DEV).to(torch.bfloat16)
    wpk = ops.pack_conv_weight(rand_w(co, ci, k, 2))
    gc = torch.Generator().manual_seed(3)
    gamma, beta = (torch.rand(co, generator=gc) + 0.5).to(DEV), (torch.rand(co, generator=gc) - 0.5).to(DEV)
    rm0, rv0 = (0.1 * torch.randn(co, generator=gc)).to(DEV), (torch.rand(co, generator=gc) + 0.5).to(DEV)
    ho, wo = ops.conv_out_hw(h, w, k, s)
    mom, eps = 0.03, 1e-3

    def run(updates):
        rm, rv = rm0.clone(), rv0.clone()
        nbt = torch.full((), 5, dtype=torch.long, device=DEV)
        raw = View.empty(n, ho, wo, co, DEV)
        ss = torch.full((2, 2, co), float("nan"), device=DEV)
        mi = torch.full((2, 2, co), float("nan"), device=DEV)
        partials = torch.empty((ops.conv_stat_rows(), 4 * co), device=DEV)
        sync = torch.zeros(2, dtype=torch.int32, device=DEV)
        ops.conv2d(View(xb), wpk, raw, k, s, ops.SY_CONV_RAW, partials=partials, bn=[(gamma, beta, rm, rv, nbt, 0)],
                   momentum=mom, eps=eps, scale_shift=ss, sync=sync, mean_invstd=mi, tile_mode=tile_mode, tile_bn=tile_bn,
                   stat_updates=updates)
        torch.cuda.synchronize()
        assert sync.tolist() == [0, 0]
        return raw.buf, ss[:, 0], mi[:, 0], rm, rv, int(nbt)

    raw1, ss1, mi1, rm1, rv1, nbt1 = run(1)
    raw2, ss2, mi2, rm2, rv2, nbt2 = run(2)
    assert torch.equal(raw1, raw2) and torch.equal(ss1, ss2) and torch.equal(mi1, mi2)
    assert (nbt1, nbt2) == (6, 7)
    # fp64 double update of the kernel's own published batch statistics (mean; variance from invstd = 1 / sqrt(var + eps))
    cnt = n * ho * wo
    mean = mi2[0].double()
    var = (1.0 / mi2[1].double() ** 2 - eps).clamp_min(0) * (cnt / (cnt - 1))
    want_m, want_v = rm0.double(), rv0.double()
    for _ in range(2):
        want_m = (1 - mom) * want_m + mom * mean
        want_v = (1 - mom) * want_v + mom * var
    for got, want, what in ((rm2, want_m, "running_mean"), (rv2, want_v, "running_var")):
        err = (got.double() - want).abs()
        assert bool((err <= 1e-6 * want.abs() + 1e-6 * float(want.abs().max())).all()), f"{what}: max err {float(err.max()):.3e}"
    # one update from the same statistics is what stat_updates = 1 wrote
    err1 = (rm1.double() - ((1 - mom) * rm0.double() + mom * mean)).abs()
    assert bool((err1 <= 1e-6 * float(rm1.abs().max())).all())


# ------------------------------------------------------------------------------------------------ 2. single pass vs duplication
def _grads_and_buffers(m):
    return ({k: p.grad.detach().float().clone() for k, p in m.named_parameters()},
            {k: v.detach().clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k})


def test_single_pass_equals_duplicated_pair_s_600x960():
    """StreamYOLO-s still model at 600 x 960, B = 2, fresh state each time: ``x`` [B, 3, H, W] (one backbone pass, running
    updates applied twice) against ``cat(x, x)`` [B, 6, H, W] (the reference's duplicated pair, two statistics groups).
    Same arithmetic, different fp32 reduction orders and bf16 rounding points, which a train-mode BatchNorm net on
    synthetic weights amplifies: the yardstick is the product's own rounding-noise floor, the duplicated run with its input
    nudged by 1e-6.  Losses within that floor (the bar of tests/test_gpu_model.py); every backbone / PAFPN conv's weight
    gradient at least as close to the duplicated run's as the nudged run is (measured on an H100: cosine >= 0.946, median
    0.972, against a floor of 0.711 / 0.740); running statistics within 2e-3."""
    x, labels = still_batch(2, 600, 960)
    x6 = torch.cat([x, x], 1)
    runs = {}
    for name, inp in (("single", x), ("pair", x6), ("pair_nudged", x6 * (1 + 1e-6))):
        m = build_still(0.33, 0.50)
        loss = backward.forward_backward(m, inp, labels)
        torch.cuda.synchronize()
        runs[name] = (np.array([float(loss[k]) for k in ORDER]),) + _grads_and_buffers(m)
    got, want, pert = runs["single"][0], runs["pair"][0], runs["pair_nudged"][0]
    floor = np.abs(pert - want)
    tol = 2.0 * floor + 5e-2 * np.abs(want) + 5e-3
    assert (np.abs(got - want)[:5] <= tol[:5]).all(), f"losses {got} vs duplicated {want} (noise floor {floor})"
    assert abs(got[5] - want[5]) <= 0.15 + 2.0 * floor[5]

    def cos(a, b):
        a, b = a.flatten().double(), b.flatten().double()
        return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-30))

    gs, gp, gn = runs["single"][1], runs["pair"][1], runs["pair_nudged"][1]
    cs, bad = [], []
    for k in gs:
        if k.startswith("backbone.") and k.endswith("conv.weight"):
            assert torch.isfinite(gs[k]).all(), k
            c, c_floor = cos(gs[k], gp[k]), cos(gn[k], gp[k])
            cs.append(c)
            if 1.0 - c > 1.0 - c_floor:
                bad.append(f"{k}: cosine {c:.5f}, noise floor {c_floor:.5f}")
    assert not bad, "\n".join(bad)
    assert min(cs) >= 0.9 and float(np.median(cs)) >= 0.95, (min(cs), float(np.median(cs)))
    bs, bp = runs["single"][2], runs["pair"][2]
    for k in bs:
        if k.endswith("num_batches_tracked"):
            assert int(bs[k]) == int(bp[k]) == (1 if k.startswith("head.") else 2), k
        else:
            assert torch.allclose(bs[k], bp[k], rtol=2e-3, atol=2e-3 * float(bp[k].abs().max())), k


# ------------------------------------------------------------------------------------------------ 3. the walk in situ
def test_walk_in_situ_every_conv_backward_still():
    """tests/test_gpu_train.py::test_walk_in_situ_every_conv_backward on the still model: every recorded conv's
    BatchNorm+SiLU, weight and data gradient against float64 torch on the very tensors the kernels read, on a NaN-poisoned
    arena -- including the DFP region whose residual half is deferred and whose jian data gradients then write it whole."""
    from test_gpu_parity_bwd import run_walk_checked
    c = CASES["tiny_120x160"]
    x, labels = still_batch(c["B"], c["H"], c["W"])
    m = build_still(c["depth"], c["width"])
    seen = run_walk_checked(m, x, labels)
    assert len(seen) == 77 - 8 - 3 + 3 - 1, len(seen)
    assert int(m.state_dict()["backbone.backbone.dark3.0.bn.num_batches_tracked"]) == 2


# ------------------------------------------------------------------------------------------------ 4. the training loops
def test_reference_trainer_sequence_with_grad_scaler():
    """/root/reference/exps/train_utils/trainer.py's step on the still cfg's model: ``outputs = model(inps, targets)``,
    ``scaler.scale(loss).backward()``, ``scaler.step(optimizer)``; the gradients autograd hands the optimiser are those of
    the explicit walk, times the scale."""
    c = CASES["tiny_120x160"]
    x, labels = still_batch(c["B"], c["H"], c["W"])
    ref = build_still(c["depth"], c["width"])
    backward.forward_backward(ref, x, labels)
    m = build_still(c["depth"], c["width"])
    opt = train.build_optimizer(m, lr=1e-4)
    scaler = torch.amp.GradScaler("cuda", init_scale=256.0)
    w0 = m.backbone.backbone.dark3[0].conv.weight.detach().clone()
    out = m(x, labels)
    assert out["total_loss"].requires_grad
    scaler.scale(out["total_loss"]).backward()
    for (k, p), q in zip(m.named_parameters(), ref.parameters()):
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        assert torch.allclose(p.grad, 256.0 * q.grad, rtol=1e-5, atol=1e-6 * float(q.grad.abs().max()) * 256.0 + 1e-12), k
    scaler.step(opt)
    scaler.update()
    assert not torch.equal(w0, m.backbone.backbone.dark3[0].conv.weight)


def test_still_trainer_graph_replay_equals_eager_steps():
    """Trainer.capture / replay on 3-channel batches and one label tensor: replays reproduce the eager steps bit for bit,
    and training on a fixed batch brings the loss down."""
    c = CASES["tiny_120x160"]
    x, labels = still_batch(c["B"], c["H"], c["W"])
    a = build_still(c["depth"], c["width"])
    ta = train.Trainer(a, lr=1e-4)
    n = 8
    want = [float(ta.step(x, labels)["total_loss"]) for _ in range(n)]
    b = build_still(c["depth"], c["width"])
    tb = train.Trainer(b, lr=1e-4)
    xs, ls = x.clone(), labels.clone()
    tb.capture(xs, ls)                                   # runs step 1 eagerly (warm-up), then captures
    got = [float(tb.replay()["total_loss"]) for _ in range(n - 1)]
    torch.cuda.synchronize()
    assert got == want[1:], (got, want)
    assert torch.equal(ta.fs.state, tb.fs.state) and torch.equal(ta.fs.ema, tb.fs.ema) and torch.equal(ta.fs.mom, tb.fs.mom)
    assert np.isfinite(want).all() and min(want[n // 2:]) < want[0], want
    assert int(b.state_dict()["backbone.backbone.stem.conv.bn.num_batches_tracked"]) == 2 * n
