"""GPU: the training-step kernels and their assembly (SURVEY section 8: rows a19, f3, f4).

  * sy_pack_conv_weight        bit-exact against the ATen permute + cast it replaces (forward, data-gradient and stem layouts)
  * sy_sgd_nesterov_ema_step   bit-for-bit against torch.optim.SGD (momentum, nesterov, weight-decay groups) + [yolox] ModelEMA
                               arithmetic in fp32 on the same device
  * sy_resize_bilinear / sy_scale_labels   Exp.preprocess (F.interpolate bilinear, align_corners=False) within 1e-5
  * train.Trainer              the flat-state step: its gradients are the very tensors the stand-alone walk produces, a few steps
                               reduce the loss, BatchNorm buffers and the EMA copy move
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import backward  # noqa: E402
from test_gpu_model import build_product  # noqa: E402


@pytest.mark.parametrize("shape", [(64, 32, 3, 3), (128, 64, 1, 1), (24, 8, 3, 3), (256, 1024, 1, 1)])
def test_pack_conv_weight_exact(shape):
    w = torch.randn(shape, device="cuda")
    o, i, kh, kw = shape
    want = w.permute(0, 2, 3, 1).reshape(o, kh * kw, i).to(torch.bfloat16).contiguous()
    assert torch.equal(ops.pack_conv_weight(w), want)
    wd = w.flip(2, 3).transpose(0, 1).contiguous()
    want_d = wd.permute(0, 2, 3, 1).reshape(i, kh * kw, o).to(torch.bfloat16).contiguous()
    assert torch.equal(ops.pack_conv_weight_dgrad(w), want_d)
    w2 = torch.randn(shape, device="cuda")
    assert torch.equal(ops.pack_conv_weight(w, w2), torch.cat([want, ops.pack_conv_weight(w2)], 0))
    pair = torch.cat([w, w2], 0)
    want_p = pair.flip(2, 3).transpose(0, 1).contiguous().permute(0, 2, 3, 1).reshape(i, kh * kw, 2 * o).to(torch.bfloat16)
    assert torch.equal(ops.pack_conv_weight_dgrad(w, w2), want_p.contiguous())


def test_pack_stem_weight_exact():
    w = torch.randn((64, 12, 3, 3), device="cuda")
    p = torch.zeros((64, 3, 4, 16), dtype=torch.bfloat16, device="cuda")
    p[:, :, :3, :12] = w.permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(ops.pack_stem_weight(w), p.reshape(64, 3, 64))


@pytest.mark.parametrize("nesterov", [True, False])
def test_fused_sgd_ema_bit_exact(nesterov):
    """Three steps on random state: parameters, momentum buffers and the EMA copy must be bit-identical to torch.optim.SGD
    (two groups: no decay | weight decay 5e-4) + the ModelEMA update, all in fp32 on the GPU."""
    torch.manual_seed(0)
    n_a, n_b, n_buf = 1000, 50000, 300
    n_param = n_a + n_b
    state = torch.randn(n_param + n_buf, device="cuda")
    mom = torch.zeros(n_param, device="cuda")
    ema = state.clone()
    pa = torch.nn.Parameter(state[:n_a].clone())
    pb = torch.nn.Parameter(state[n_a:n_param].clone())
    opt = torch.optim.SGD([pa], lr=0.0125, momentum=0.9, nesterov=nesterov)
    opt.add_param_group({"params": [pb], "weight_decay": 5e-4})
    ref_ema = state.clone()
    for it in range(1, 4):
        g = torch.randn(n_param, device="cuda") * 64.0          # a scaled gradient (GradScaler)
        inv = 1.0 / 64.0
        d = 0.9998 * (1 - math.exp(-it / 2000))
        state[n_param:] += 0.01                                 # the BatchNorm buffers move with the forward
        ops.sgd_nesterov_ema_step(state, g, mom, ema, n_param, n_a, 0.0125, 0.9, 5e-4, inv_scale=inv, nesterov=nesterov,
                                  ema_decay=d)
        gu = g * inv                                            # GradScaler.unscale_
        pa.grad, pb.grad = gu[:n_a].clone(), gu[n_a:].clone()
        opt.step()
        msd = torch.cat([pa.detach(), pb.detach(), state[n_param:]])
        ref_ema.mul_(d).add_((1.0 - d) * msd)
        torch.cuda.synchronize()
        assert torch.equal(state[:n_a], pa.detach()) and torch.equal(state[n_a:n_param], pb.detach()), f"step {it}"
        assert torch.equal(mom[n_a:], opt.state[pb]["momentum_buffer"])
        assert torch.equal(ema, ref_ema), f"ema step {it}"
    # found_inf skips the update
    before = state.clone()
    ops.sgd_nesterov_ema_step(state, g, mom, ema, n_param, n_a, 0.0125, found_inf=torch.ones(1, device="cuda"))
    assert torch.equal(before, state)


@pytest.mark.parametrize("size", [(480, 768), (640, 1024), (600, 960), (333, 517)])
def test_resize_bilinear_matches_interpolate(size):
    x = torch.rand((2, 6, 600, 960), device="cuda") * 255
    got = ops.resize_bilinear(x, size)
    want = F.interpolate(x, size=size, mode="bilinear", align_corners=False)
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-3), float((got - want).abs().max())
    cpu = F.interpolate(x.cpu(), size=size, mode="bilinear", align_corners=False)
    assert torch.allclose(got.cpu(), cpu, rtol=1e-5, atol=1e-3)
    lab = torch.rand((2, 120, 5), device="cuda") * 100
    want_l = lab.clone()
    sx, sy = size[1] / 960, size[0] / 600
    want_l[..., 1::2] = want_l[..., 1::2] * sx
    want_l[..., 2::2] = want_l[..., 2::2] * sy
    assert torch.equal(ops.scale_labels_(lab, sx, sy), want_l)


def test_trainer_flat_gradients_equal_standalone_walk():
    """FlatSink (kernels write into the flat buffer, accumulate flags from first-touch tracking) against TensorSink (fresh
    tensors): the same kernels on the same inputs -- every parameter gradient must be bit-identical."""
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"]).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(c["B"], c["H"], c["W"]))
    a = build_product(c["depth"], c["width"]).train()
    backward.forward_backward(a, x, tg)
    b = build_product(c["depth"], c["width"]).train()
    tr = train.Trainer(b, lr=1e-3)
    tr.forward_backward(x, tg)
    torch.cuda.synchronize()
    for (k, p), q in zip(a.named_parameters(), b.parameters()):
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        assert torch.equal(p.grad, q.grad), k
    assert sum(e - s for s, e in tr.sink.launched) == tr.fs.n_param


def test_trainer_steps_reduce_the_loss_on_gpu():
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"]).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(c["B"], c["H"], c["W"]))
    m = build_product(c["depth"], c["width"]).train()
    w0 = m.backbone.backbone.dark3[0].conv.weight.detach().clone()
    tr = train.Trainer(m, lr=2e-4)
    losses = [float(tr.step(x, tg)["total_loss"]) for _ in range(5)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert not torch.equal(w0, m.backbone.backbone.dark3[0].conv.weight)
    assert int(m.state_dict()["backbone.jian0.bn.num_batches_tracked"]) == 10
    esd = tr.ema_state_dict()
    k = "backbone.backbone.dark3.0.conv.weight"
    assert torch.isfinite(esd[k]).all() and not torch.equal(esd[k], m.state_dict()[k])
    # the reference trainer's call sequence on the same model class: loss with a grad_fn, .backward(), torch optimizer
    m2 = build_product(c["depth"], c["width"]).train()
    opt = train.build_optimizer(m2, lr=2e-4)
    l0 = None
    for _ in range(3):
        opt.zero_grad()
        out = m2(x, tg)
        assert out["total_loss"].requires_grad
        out["total_loss"].backward()
        opt.step()
        l0 = l0 or float(out["total_loss"])
    assert float(out["total_loss"]) < l0


def test_walk_in_situ_every_conv_backward():
    """The assembled backward on the GPU, checked op by op INSIDE the walk: for every recorded BaseConv launch (73 modules,
    DFP jian twice) the BatchNorm+SiLU gradient, the weight gradient and the (accumulated) data gradient the kernels produce
    are compared with float64 torch on the very tensors the kernels read (the gradient buffer as it stood, the saved raw
    output / statistics, the bf16 weights).  Identical inputs per step: no chaos amplification, so bf16-ulp and fp32-reduction
    tolerances hold (the checker and its bars: tests/test_gpu_parity_bwd.py, which runs it at the benchmarked sizes).
    Together with the exact routing test on CPU (tests/test_cpu_backward.py) this pins the walk on hardware."""
    from test_gpu_parity_bwd import run_walk_checked
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"]).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(c["B"], c["H"], c["W"]))
    m = build_product(c["depth"], c["width"]).train()
    seen = run_walk_checked(m, x, tg)
    # 77 BaseConvs: 8 CSP conv2 ride with their conv1, 3 head reg towers with their cls twin, jian x2, the stem has no dx
    assert len(seen) == 77 - 8 - 3 + 3 - 1, len(seen)


def test_trainer_graph_replay_equals_eager_steps():
    """The whole step (recording forward, walk, weight re-pack, fused optimiser + EMA) captured as one CUDA graph: replays
    must reproduce the eager steps bit for bit -- including the EMA decay ramp and the learning rate, which reach the
    captured kernel through the device-side hyper-parameter block."""
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"]).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(c["B"], c["H"], c["W"]))
    a = build_product(c["depth"], c["width"]).train()
    ta = train.Trainer(a, lr=2e-4)
    lrs = [2e-4, 1.5e-4, 1e-4]
    want = [float(ta.step(x, tg, lr=lr)["total_loss"]) for lr in lrs]
    b = build_product(c["depth"], c["width"]).train()
    tb = train.Trainer(b, lr=lrs[0])
    xs, ts = x.clone(), tuple(t.clone() for t in tg)
    tb.capture(xs, ts)                                   # runs step 1 eagerly (warm-up) with lr[0], then captures
    got = [float(tb.replay(lr=lr)["total_loss"]) for lr in lrs[1:]]
    torch.cuda.synchronize()
    assert got == want[1:], (got, want)
    assert torch.equal(ta.fs.state, tb.fs.state) and torch.equal(ta.fs.ema, tb.fs.ema) and torch.equal(ta.fs.mom, tb.fs.mom)


def test_pack_batch_equals_single_packs():
    """sy_pack_conv_weights_batch (every operand of a model in ONE launch) against the per-parameter launches, bit for bit:
    forward layout, pair concatenation, data-gradient layout with pitch / column offset, the Focus-stem layout."""
    g = torch.Generator().manual_seed(5)
    ws = [torch.randn(s, generator=g).cuda() for s in ((64, 32, 3, 3), (24, 64, 1, 1), (40, 64, 1, 1), (16, 12, 3, 3), (128, 128, 3, 3))]
    pb = ops.PackBatch(torch.device("cuda"))
    f0 = torch.empty((64, 9, 32), dtype=torch.bfloat16, device="cuda")
    d0 = torch.empty((32, 9, 64), dtype=torch.bfloat16, device="cuda")
    pair_f = torch.empty((64, 1, 64), dtype=torch.bfloat16, device="cuda")
    pair_d = torch.empty((64, 1, 64), dtype=torch.bfloat16, device="cuda")
    stem = torch.empty((16, 3, 64), dtype=torch.bfloat16, device="cuda")
    f4 = torch.empty((128, 9, 128), dtype=torch.bfloat16, device="cuda")
    pb.add(ws[0], f0, 0)
    pb.add(ws[0], d0, 1, out_pitch=64, co_offset=0)
    pb.add(ws[1], pair_f[0:24], 0)
    pb.add(ws[2], pair_f[24:64], 0)
    pb.add(ws[1], pair_d, 1, out_pitch=64, co_offset=0)
    pb.add(ws[2], pair_d, 1, out_pitch=64, co_offset=24)
    pb.add(ws[3], stem, 2)
    pb.add(ws[4], f4, 0)
    pb.run()
    torch.cuda.synchronize()
    assert torch.equal(f0, ops.pack_conv_weight(ws[0])) and torch.equal(d0, ops.pack_conv_weight_dgrad(ws[0]))
    assert torch.equal(pair_f, ops.pack_conv_weight(ws[1], ws[2])) and torch.equal(pair_d, ops.pack_conv_weight_dgrad(ws[1], ws[2]))
    assert torch.equal(stem, ops.pack_stem_weight(ws[3])) and torch.equal(f4, ops.pack_conv_weight(ws[4]))
    # ragged tiles (the launch works in 64 x 32 channel tiles) and a stem with more than 64 outputs
    for shape in ((96, 80, 3, 3), (200, 24, 3, 3), (520, 264, 1, 1), (8, 8, 3, 3)):
        w = torch.randn(shape, generator=g).cuda()
        o, i, kh, kw = shape
        f = torch.full((o, kh * kw, i), 7.0, dtype=torch.bfloat16, device="cuda")
        d = torch.full((i, kh * kw, o + 8), 7.0, dtype=torch.bfloat16, device="cuda")
        pb2 = ops.PackBatch(torch.device("cuda"))
        pb2.add(w, f, 0)
        pb2.add(w, d, 1, out_pitch=o + 8, co_offset=8)
        pb2.run()
        torch.cuda.synchronize()
        assert torch.equal(f, ops.pack_conv_weight(w))
        assert torch.equal(d[:, :, 8:], ops.pack_conv_weight_dgrad(w)) and (d[:, :, :8] == 7.0).all()
    w = torch.randn((80, 12, 3, 3), generator=g).cuda()
    st = torch.empty((80, 3, 64), dtype=torch.bfloat16, device="cuda")
    pb3 = ops.PackBatch(torch.device("cuda"))
    pb3.add(w, st, 2)
    pb3.run()
    torch.cuda.synchronize()
    assert torch.equal(st, ops.pack_stem_weight(w))
