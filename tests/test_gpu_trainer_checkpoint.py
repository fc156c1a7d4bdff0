"""GPU: saving and resuming the Trainer (train.Trainer.state_dict / load_state_dict) with the real kernels, eagerly and
under CUDA graphs.  Every comparison is bit for bit against a run that was not interrupted: the flat state, momentum, EMA
copy, BatchNorm buffers, ``updates`` and the losses.  Loading copies into the buffers the captured graphs read, so a
Trainer whose graphs are captured keeps replaying them after a load."""
import io
import os
import random
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from streamyolo_b200 import synth, train  # noqa: E402
from test_gpu_parity_fwd import _build  # noqa: E402
from test_multiscale_train import _Inputs, _assert_same, _snapshot  # noqa: E402

pytestmark = pytest.mark.gpu

INPUT = (600, 960)


def _lr(i):
    return 1e-4 * (1 + 0.1 * i)


def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf)


def test_state_dict_continues_bit_exactly_s():
    """StreamYOLO-s, 4 pairs at 600x960, eager: 5 steps == 2 steps, save, a fresh model + Trainer, load, 3 steps"""
    def batch(i):
        return (synth.synth_frames(4, *INPUT, seed=200 + i).cuda(),
                tuple(t.cuda() for t in synth.synth_labels(4, *INPUT, seed=300 + i)))

    a = train.Trainer(_build("s"), lr=1e-4)
    want = [float(a.step(*batch(i), lr=_lr(i))["total_loss"]) for i in range(5)]
    b = train.Trainer(_build("s"), lr=1e-4)
    for i in range(2):
        b.step(*batch(i), lr=_lr(i))
    sd = _roundtrip(b.state_dict())
    del b
    c = train.Trainer(_build("s"), lr=1e-4)
    c.load_state_dict(sd)
    got = [float(c.step(*batch(i), lr=_lr(i))["total_loss"]) for i in range(2, 5)]
    torch.cuda.synchronize()
    assert got == want[2:], (got, want)
    _assert_same(_snapshot(c), _snapshot(a), "resumed eager run")


def test_load_into_a_captured_trainer_one_size():
    """StreamYOLO-s, 2 pairs, one captured size.  A replays 5 steps.  B replays 2, saves, replays 2 more steps on other
    data (so the load has something to undo), loads the saved state into the same Trainer, whose graph stays captured,
    and replays the last 3: B ends where A ends."""
    dev = torch.device("cuda")
    size = [INPUT]
    inp_a = _Inputs(2, INPUT, False, dev, size)
    a = train.Trainer(_build("s"), lr=1e-4)
    a.capture_sizes(size, inp_a.make_inputs, inp_a.prologue)
    want = []
    for i in range(5):
        inp_a.load(100 + i)
        want.append(float(a.replay_size(INPUT, lr=_lr(i))["total_loss"]))
    inp_b = _Inputs(2, INPUT, False, dev, size)
    b = train.Trainer(_build("s"), lr=1e-4)
    b.capture_sizes(size, inp_b.make_inputs, inp_b.prologue)
    for i in range(2):
        inp_b.load(100 + i)
        b.replay_size(INPUT, lr=_lr(i))
    sd = _roundtrip(b.state_dict())
    for i in range(2):
        inp_b.load(900 + i)
        b.replay_size(INPUT, lr=1e-3)
    b.load_state_dict(sd)
    got = []
    for i in range(2, 5):
        inp_b.load(100 + i)
        got.append(float(b.replay_size(INPUT, lr=_lr(i))["total_loss"]))
    torch.cuda.synchronize()
    assert got == want[2:], (got, want)
    _assert_same(_snapshot(b), _snapshot(a), "load into a captured Trainer")


def test_resume_multiscale_graphs_in_a_fresh_trainer():
    """StreamYOLO-s, 2 pairs, three of the cfg's multi-scale sizes interleaved over 8 replays.  The interrupted run stops
    after step 4 and saves; a fresh model + Trainer loads the state, captures the sizes afresh (capture_sizes leaves the
    loaded state as it found it) and replays steps 5-8: same losses and same final state as the uninterrupted run."""
    dev = torch.device("cuda")
    all_sizes = train.multiscale_sizes()
    sizes = [all_sizes[0], INPUT, all_sizes[-2]]             # 496x800, 600x960, 688x1120
    rng = random.Random(5)
    seq = sizes + [rng.choice(sizes) for _ in range(5)]
    assert len(set(seq[4:])) >= 2

    def run(tr, inp, steps):
        out = []
        for i in steps:
            inp.load(100 + i)
            out.append(float(tr.replay_size(seq[i], lr=_lr(i))["total_loss"]))
        return out

    inp = _Inputs(2, INPUT, False, dev, sizes)
    a = train.Trainer(_build("s"), lr=1e-4)
    a.capture_sizes(sizes, inp.make_inputs, inp.prologue)
    want = run(a, inp, range(8))
    inp_b = _Inputs(2, INPUT, False, dev, sizes)
    b = train.Trainer(_build("s"), lr=1e-4)
    b.capture_sizes(sizes, inp_b.make_inputs, inp_b.prologue)
    run(b, inp_b, range(4))
    sd = _roundtrip(b.state_dict())
    del b, inp_b
    inp_c = _Inputs(2, INPUT, False, dev, sizes)
    c = train.Trainer(_build("s"), lr=1e-4)
    c.load_state_dict(sd)
    c.capture_sizes(sizes, inp_c.make_inputs, inp_c.prologue)
    got = run(c, inp_c, range(4, 8))
    torch.cuda.synchronize()
    assert got == want[4:], (seq, got, want)
    _assert_same(_snapshot(c), _snapshot(a), "resumed multi-scale run")
