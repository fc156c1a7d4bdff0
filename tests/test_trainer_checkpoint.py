"""CPU: the Trainer's checkpoint surface (streamyolo_b200/train.py: state_dict / load_state_dict, optimizer_state_dict in
torch.optim.SGD format, reference_checkpoint / load_reference_checkpoint, all_reduce_norm) with every kernel replaced by
its torch emulation (tests/emul_ops.py).  Exact continuation is checked bit for bit; the reference's checkpoint file and
resume (exps/train_utils/double_trainer.py:285-318, 353-371) against the stock PyTorch step (train.train_step,
torch.optim.SGD, ModelEMA) at the tolerances of tests/test_cpu_train.py; the BatchNorm average over two gloo ranks against
a restatement of yolox's all_reduce_norm."""
import copy
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
import test_cpu_backward as T  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import engine  # noqa: E402

C = CASES["tiny_120x160"]
RTOL, ATOL = 1e-5, 1e-7          # test_cpu_train.py::test_trainer_step_matches_stock_pytorch_step


def _batch(i):
    return (synth.synth_frames(C["B"], C["H"], C["W"], seed=40 + i),
            synth.synth_labels(C["B"], C["H"], C["W"], seed=60 + i))


def _lr(i):
    return None if i == 4 else 2e-4 * (1 + 0.1 * i)          # the last step runs at the Trainer's own lr


def _steps(tr, idx):
    return [tr.step(*_batch(i), lr=_lr(i)) for i in idx]


def _counters(model):
    return {k: v.clone() for k, v in model.state_dict().items() if not v.dtype.is_floating_point}


def _one_storage(tensors):
    return len({t.untyped_storage().data_ptr() for t in tensors}) == 1


@pytest.mark.parametrize("use_ema", [True, False], ids=["ema", "no_ema"])
def test_state_dict_continues_bit_exactly(use_ema, tmp_path, monkeypatch):
    """5 steps == 2 steps, torch.save(state_dict()), a fresh model + Trainer, load_state_dict, 3 steps: the flat state,
    momentum, EMA copy, num_batches_tracked, updates and losses bit for bit"""
    emul_ops.install(monkeypatch, exact=True)
    a = train.Trainer(T.build_product(C), lr=2e-4, use_ema=use_ema)
    want = _steps(a, range(5))
    b = train.Trainer(T.build_product(C), lr=2e-4, use_ema=use_ema)
    _steps(b, range(2))
    path = tmp_path / "state.pt"
    torch.save(b.state_dict(), path)
    sd = torch.load(path)
    # one storage each for the weights, the momentum and the EMA copy: nothing is written twice
    assert _one_storage([t for t in sd["model"].values() if t.dtype == torch.float32])
    assert _one_storage([s["momentum_buffer"] for s in sd["optimizer"]["state"].values()])
    assert sd["ema"] is None if not use_ema else _one_storage([t for t in sd["ema"].values() if t.dtype == torch.float32])
    del b
    c = train.Trainer(T.build_product(C), lr=1.0, momentum=0.5, use_ema=use_ema)
    c.load_state_dict(sd)
    assert (c.lr, c.momentum, c.weight_decay, c.updates) == (2e-4, 0.9, 5e-4, 2)
    got = _steps(c, range(2, 5))
    assert torch.equal(c.fs.state, a.fs.state) and torch.equal(c.fs.mom, a.fs.mom)
    assert torch.equal(c.fs.ema, a.fs.ema) if use_ema else c.fs.ema is None
    ca, cc = _counters(a.model), _counters(c.model)
    assert ca.keys() == cc.keys() and all(torch.equal(ca[k], cc[k]) for k in ca)
    assert int(cc["backbone.jian0.bn.num_batches_tracked"]) == 10
    assert c.updates == a.updates == 5
    for w, g in zip(want[2:], got):
        assert w.keys() == g.keys() and all(torch.equal(w[k], g[k]) for k in w)


def test_load_keeps_buffers_and_operands_in_place(monkeypatch):
    """load_state_dict copies into the buffers a captured graph reads: the flat state, momentum, EMA copy, the modules'
    tensors and every packed conv operand keep their addresses; WEIGHT_EPOCH moves and the operands hold the loaded
    weights, registered under the key the forward looks them up with"""
    emul_ops.install(monkeypatch, exact=True)
    tr = train.Trainer(T.build_product(C), lr=2e-4)
    _steps(tr, range(2))
    snap = copy.deepcopy(tr.state_dict())
    _steps(tr, range(2, 3))
    fs = tr.fs

    def addresses():
        return ([fs.state.data_ptr(), fs.mom.data_ptr(), fs.ema.data_ptr()]
                + [t.data_ptr() for _, fwd, dg in tr._packed_groups for t in (fwd, dg) if t is not None]
                + [t.data_ptr() for t in tr.model.state_dict().values()])

    before, epoch = addresses(), engine.WEIGHT_EPOCH
    tr.load_state_dict(snap)
    assert addresses() == before and engine.WEIGHT_EPOCH > epoch
    assert tr.updates == 2
    for k, t in tr.model.state_dict().items():
        assert torch.equal(t, snap["model"][k]), k
    for i, s in snap["optimizer"]["state"].items():
        assert torch.equal(tr.optimizer_state_dict()["state"][i]["momentum_buffer"], s["momentum_buffer"]), i
    for k, t in tr.ema_state_dict().items():
        assert torch.equal(t, snap["ema"][k]), k
    for g, fwd, dg in tr._packed_groups:
        ws = [m.conv.weight for m in g]
        if dg is None:
            assert torch.equal(fwd, ops.pack_stem_weight(*ws))
            continue
        assert torch.equal(fwd, ops.pack_conv_weight(*ws)) and torch.equal(dg, ops.pack_conv_weight_dgrad(*ws))
        assert engine.packed_operand(g[0], "_pk" if len(g) == 1 else "_pk2", ws, ops.pack_conv_weight) is fwd
    state = tr.fs.state.clone()
    tr.all_reduce_norm()                                   # one process: nothing to average
    assert torch.equal(tr.fs.state, state)


def test_load_rejects_another_architecture(monkeypatch):
    emul_ops.install(monkeypatch, exact=True)
    tr = train.Trainer(T.build_product(C), lr=2e-4)
    other = train.Trainer(T.build_product(T.DEPTH_CASES["l_depth_64x96"]), lr=2e-4)
    assert other.fs.n_param != tr.fs.n_param
    before = tr.fs.state.clone()
    with pytest.raises(ValueError, match="architecture"):
        tr.load_state_dict(other.state_dict())
    with pytest.raises(ValueError, match="architecture"):
        tr.load_reference_checkpoint(other.reference_checkpoint(1), 10)
    with pytest.raises(ValueError):
        tr.load_optimizer_state_dict(other.optimizer_state_dict())
    sd = tr.state_dict()
    sd["ema"] = None
    with pytest.raises(ValueError, match="EMA"):
        tr.load_state_dict(sd)
    opt = tr.optimizer_state_dict()
    opt["param_groups"][0]["weight_decay"] = 1e-4
    with pytest.raises(ValueError, match="hyper-parameters"):
        tr.load_optimizer_state_dict(opt)
    assert torch.equal(tr.fs.state, before)


def _stock_pair(lr=2e-4):
    ref = T.build_product(C)
    return ref, train.build_optimizer(ref, lr=lr), train.ModelEMA(ref)


def _assert_momentum_close(got, want):
    assert list(got["state"]) == list(want["state"])
    for i, s in want["state"].items():
        assert got["state"][i].keys() == s.keys()
        assert torch.allclose(got["state"][i]["momentum_buffer"], s["momentum_buffer"], rtol=RTOL, atol=ATOL), i


def test_optimizer_state_dict_is_torch_sgd_format(monkeypatch):
    """optimizer_state_dict() after 3 Trainer steps == build_optimizer(...).state_dict() after 3 stock steps: keys, group
    hyper-parameters, index lists, momentum buffers; empty state before the first update; loads both ways"""
    emul_ops.install(monkeypatch, exact=True)
    x, tg = _batch(0)
    ref, opt, ema = _stock_pair()
    tr = train.Trainer(T.build_product(C), lr=2e-4)
    assert tr.optimizer_state_dict() == opt.state_dict() == {"state": {}, "param_groups": opt.state_dict()["param_groups"]}
    for _ in range(3):
        train.train_step(ref, opt, x, tg, ema)
    for _ in range(3):
        tr.step(x, tg)
    want, got = opt.state_dict(), tr.optimizer_state_dict()
    assert got.keys() == want.keys() and got["param_groups"] == want["param_groups"]
    assert [g["weight_decay"] for g in got["param_groups"]] == [0, 5e-4, 0]
    assert all(g["nesterov"] and g["momentum"] == 0.9 and g["lr"] == 2e-4 for g in got["param_groups"])
    assert len(got["state"]) == len(list(ref.parameters()))
    _assert_momentum_close(got, want)
    train.build_optimizer(T.build_product(C), lr=1.0).load_state_dict(got)
    # the reverse direction: torch's state into a fresh Trainer, exactly
    fresh = train.Trainer(T.build_product(C), lr=1.0, momentum=0.5, weight_decay=0.0)
    fresh.load_optimizer_state_dict(want)
    assert (fresh.lr, fresh.momentum, fresh.weight_decay) == (2e-4, 0.9, 5e-4)
    fresh.updates = 3
    back = fresh.optimizer_state_dict()
    assert back["param_groups"] == want["param_groups"]
    for i, s in want["state"].items():
        assert torch.equal(back["state"][i]["momentum_buffer"], s["momentum_buffer"]), i
    # no momentum_buffer: zeros (torch's first step)
    fresh.load_optimizer_state_dict(train.build_optimizer(T.build_product(C), lr=2e-4).state_dict())
    assert not bool(fresh.fs.mom.any())


def test_reference_checkpoint_resumes_like_resume_train(tmp_path, monkeypatch):
    """reference_checkpoint(3) through torch.save / torch.load, replayed with the reference's resume_train in stock PyTorch
    (model.load_state_dict(ckpt["model"]), optimizer.load_state_dict(ckpt["optimizer"]), ModelEMA(model, updates=...)):
    one train_step from there == one Trainer.step after load_reference_checkpoint on a fresh Trainer"""
    emul_ops.install(monkeypatch, exact=True)
    a = train.Trainer(T.build_product(C), lr=2e-4)
    _steps(a, range(3))
    path = tmp_path / "latest_ckpt.pth"
    torch.save(a.reference_checkpoint(3, best_ap=0.25), path)
    ckpt = torch.load(path)
    assert list(ckpt) == ["start_epoch", "model", "optimizer", "best_ap"]
    esd = a.ema_state_dict()
    assert list(ckpt["model"]) == list(esd) and all(torch.equal(ckpt["model"][k], esd[k]) for k in esd)
    updates = 3 * 10                                           # max_iter * start_epoch
    x, tg = _batch(7)
    ref = T.build_product(C)                                   # resume_train + before_train, stock PyTorch
    ref.load_state_dict(ckpt["model"])
    opt = train.build_optimizer(ref, lr=0.01)
    opt.load_state_dict(ckpt["optimizer"])
    ema = train.ModelEMA(ref, updates=updates)
    want = train.train_step(ref, opt, x, tg, ema)
    tr = train.Trainer(T.build_product(C), lr=0.01)
    assert tr.load_reference_checkpoint(torch.load(path), updates) == (3, 0.25)
    assert tr.updates == updates and tr.lr == 2e-4
    got = tr.step(x, tg)
    assert abs(float(got["total_loss"]) - float(want["total_loss"])) <= 1e-5 * abs(float(want["total_loss"]))
    for (k, p), q in zip(tr.model.named_parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=RTOL, atol=ATOL), k
    esd, rsd = tr.ema_state_dict(), ema.ema.state_dict()
    for k in rsd:
        if rsd[k].dtype.is_floating_point:
            assert torch.allclose(esd[k], rsd[k], rtol=RTOL, atol=ATOL), k
    _assert_momentum_close(tr.optimizer_state_dict(), opt.state_dict())


def test_stock_checkpoint_loads_into_trainer(tmp_path, monkeypatch):
    """a file the reference's save_ckpt writes (EMA weights, torch.optim.SGD state) loads into a Trainer exactly"""
    emul_ops.install(monkeypatch, exact=True)
    ref, opt, ema = _stock_pair()
    for i in range(2):
        train.train_step(ref, opt, *_batch(i), ema)
    path = tmp_path / "latest_ckpt.pth"
    torch.save({"start_epoch": 1, "model": ema.ema.state_dict(), "optimizer": opt.state_dict(), "best_ap": 0.5}, path)
    tr = train.Trainer(T.build_product(C), lr=1.0)
    assert tr.load_reference_checkpoint(torch.load(path), 20) == (1, 0.5)
    esd = ema.ema.state_dict()
    for k, t in tr.model.state_dict().items():
        assert torch.equal(t, esd[k]), k
    assert torch.equal(tr.fs.ema, tr.fs.state)               # the EMA restarts from the loaded weights
    got, want = tr.optimizer_state_dict(), opt.state_dict()
    assert got["param_groups"] == want["param_groups"]
    for i, s in want["state"].items():
        assert torch.equal(got["state"][i]["momentum_buffer"], s["momentum_buffer"]), i


NORM_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
from collections import OrderedDict
import torch
import torch.distributed as dist
import emul_ops, test_cpu_backward as T
from oracle.make_golden import CASES
from streamyolo_b200 import dist as d, synth, train


class MP:
    def setattr(self, o, n, v): setattr(o, n, v)
    def setitem(self, dct, k, v): dct[k] = v


def yolox_all_reduce_norm(model):
    # [yolox 0.3.0] yolox/utils/allreduce_norm.py: every BatchNorm state entry, flattened into one tensor, summed over
    # the ranks, divided by the world size; returns what all_reduce_norm loads back into the model
    states = OrderedDict()
    for name, child in model.named_modules():
        if isinstance(child, torch.nn.BatchNorm2d):
            for k, v in child.state_dict().items():
                states[name + "." + k] = v
    keys = list(states)
    flat = torch.cat([states[k].flatten() for k in keys])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat /= dist.get_world_size()
    parts = torch.split(flat, [states[k].numel() for k in keys])
    return {k: p.reshape(states[k].shape).to(states[k].dtype) for k, p in zip(keys, parts)}


rank, local, world = d.init("gloo")
emul_ops.install(MP(), exact=True)
c = CASES["tiny_120x160"]
x = synth.synth_frames(4, c["H"], c["W"])
fut, cur = synth.synth_labels(4, c["H"], c["W"])
lo, hi = d.shard_pairs(4, world, rank)
model = T.build_product(c)
tr = train.Trainer(model, lr=1e-3, bucket_bytes=64 << 10)
for _ in range(2):
    tr.step(x[lo:hi], (fut[lo:hi], cur[lo:hi]))
want = yolox_all_reduce_norm(model)
k = "backbone.backbone.dark3.0.bn.running_mean"
mine = model.state_dict()[k].clone()
other = [torch.empty_like(mine) for _ in range(world)]
dist.all_gather(other, mine)
assert not torch.equal(other[0], other[1])                     # different shards: different statistics
n = tr.fs.n_param
params, mom, ema = tr.fs.state[:n].clone(), tr.fs.mom.clone(), tr.fs.ema.clone()
tr.all_reduce_norm()
sd = model.state_dict()
assert len(want) == 5 * sum(isinstance(m, torch.nn.BatchNorm2d) for m in model.modules())
for key, v in want.items():
    assert torch.equal(sd[key], v), key
assert torch.equal(sd[k], (other[0] + other[1]) / 2)
assert torch.equal(tr.fs.state[:n], params) and torch.equal(tr.fs.mom, mom) and torch.equal(tr.fs.ema, ema)
print("ok", rank)
"""


def test_all_reduce_norm_gloo_world2(tmp_path):
    """two gloo ranks step on different shards, so their BatchNorm statistics differ; after Trainer.all_reduce_norm()
    both hold exactly what yolox's all_reduce_norm computes, (stats_0 + stats_1) / 2, and the parameters, momentum and EMA
    copy are untouched"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "norm.py"
    script.write_text(NORM_WORKER)
    port = 29400 + os.getpid() % 90
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                   OMP_NUM_THREADS="4")
        procs.append(subprocess.Popen([sys.executable, str(script), root], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(o[-3000:] for o in outs)
