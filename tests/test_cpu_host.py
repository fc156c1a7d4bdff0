"""CPU: the C-ABI library loads and exports every symbol the header declares, host-side logic,
state_dict parity of the module mirror, loud failure without a GPU, and the world_size-2
(gloo) sharding / timing-reduction path of the benchmark."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from streamyolo_b200 import dist as sydist
from streamyolo_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def lib():
    from streamyolo_b200.build import build
    build()
    return ops.load_library()


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "streamyolo_sm100.h")).read()
    declared = set(re.findall(r"\b(sy_[a-z0-9_]+)\s*\(", hdr)) - {"sy_stream_t"}
    assert declared == set(ops.EXPORTED_SYMBOLS), declared ^ set(ops.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.sy_version() >= 100


def test_host_logic_no_gpu(lib):
    assert lib.sy_conv_stat_rows() >= 1          # one statistics row per persistent CTA (SM count; 132 on H100)
    assert lib.sy_stats_num_partials(4, 1000) == 8
    assert lib.sy_tal_loss_workspace_bytes(8, 11850, 120, 8) > 2 * 8 * 120 * 11850 * 4


def test_compute_fails_loudly_without_gpu(lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    v = ops.View(torch.zeros((1, 4, 4, 8), dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.copy(v, v)


@pytest.mark.parametrize("tag,dw", [("s", (0.33, 0.5)), ("m", (0.67, 0.75)), ("l", (1.0, 1.0))])
def test_module_mirror_state_dict(tag, dw):
    from streamyolo_b200.model import DFPPAFPN, TALHead, YOLOX
    g = np.load(os.path.join(GOLD, "state_shapes.npz"))
    m = YOLOX(DFPPAFPN(dw[0], dw[1], in_channels=[256, 512, 1024]), TALHead(8, dw[1], in_channels=[256, 512, 1024]))
    sd = m.state_dict()
    assert list(sd) == g[tag + "_keys"].tolist()                       # same keys, same order as the reference
    assert ["x".join(map(str, v.shape)) for v in sd.values()] == g[tag + "_shapes"].tolist()
    assert sum(p.numel() for p in m.parameters()) == int(g[tag + "_nparams"])
    # init_yolo / initialize_biases hooks of cfgs/*.py:40-54 work on the mirror
    n_bn = sum(isinstance(x, torch.nn.BatchNorm2d) for x in m.modules())
    assert n_bn == {"s": 77, "m": 101, "l": 125}[tag]
    m.head.initialize_biases(1e-2)
    assert abs(float(m.head.cls_preds[0].bias[0]) + 4.59512) < 1e-4
    assert m.head.use_l1 is False and m.head.decode_in_inference is True and m.head.n_anchors == 1


def test_shard_pairs():
    for gb, w in [(32, 8), (64, 8), (8, 1), (10, 4), (3, 2)]:
        spans = [sydist.shard_pairs(gb, w, r) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == gb
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        sizes = [b - a for a, b in spans]
        assert max(sizes) - min(sizes) <= 1


WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1])
import torch
from streamyolo_b200 import dist as d
rank, local, world = d.init("gloo")
a, b = d.shard_pairs(10, world, rank)
d.barrier()
t = d.max_over_ranks(1.0 + rank)
n = d.sum_over_ranks(b - a)
assert t == float(world) and n == 10.0, (t, n)
print("ok", rank)
"""


def test_gloo_world2(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(WORKER)
    port = 29600 + os.getpid() % 300
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs


def test_dropin_aliases():
    """cfgs/*.py: `from exps.model.yolox import YOLOX` etc. must resolve to this package's classes after install()."""
    code = ("import streamyolo_b200.dropin as d; d.install();"
            "from exps.model.yolox import YOLOX; from exps.model.dfp_pafpn import DFPPAFPN;"
            "from exps.model.tal_head import TALHead; from exps.model.darknet import CSPDarknet;"
            "from exps.model.pipe_head import PIPEHead; assert issubclass(PIPEHead, TALHead);"
            "import streamyolo_b200.model as m; assert YOLOX is m.YOLOX and TALHead is m.TALHead; print('ok')")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr


def test_struct_layouts_match_header(tmp_path):
    """Every descriptor struct of include/streamyolo_sm100.h, compiled by gcc, has the size and the field offsets of its
    ctypes twin in streamyolo_b200/ops.py (a silent mismatch would corrupt kernel arguments)."""
    import ctypes
    import re
    import shutil
    from streamyolo_b200 import ops
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    names = [n for n in dir(ops) if n.startswith("Sy") and isinstance(getattr(ops, n), type)
             and issubclass(getattr(ops, n), ctypes.Structure)]
    header = open(os.path.join(ROOT, "include", "streamyolo_sm100.h")).read()
    assert set(names) == set(re.findall(r"\}\s*(Sy\w+)\s*;", header)), "ctypes stubs and header structs differ"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "streamyolo_sm100.h"', "int main(void) {"]
    for n in names:
        lines.append(f'  printf("{n} size %zu\\n", sizeof({n}));')
        for f, _ in getattr(ops, n)._fields_:
            lines.append(f'  printf("{n} {f} %zu\\n", offsetof({n}, {f}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.split("\n")
    for line in filter(None, out):
        n, f, v = line.split()
        cls = getattr(ops, n)
        want = ctypes.sizeof(cls) if f == "size" else getattr(cls, f).offset
        assert int(v) == want, f"{n}.{f}: header {v}, ctypes {want}"


def test_conv_tiling_plan_and_overrides_without_gpu():
    """sy_conv2d_plan is host-only: the tiling decisions of the tensor-core conv can be inspected (and are pinned here for the
    layers that motivated them) without a device, with and without the tile_mode / tile_bn overrides; out-of-range
    overrides are rejected.  132 SMs (an H100 SXM) are assumed when no GPU is present."""
    p = ops.conv2d_plan(16, 38, 60, 256, 256, 3, 1)          # linear tiles: 285 x 2 tiles = 5 rounds
    assert (p["mode"], p["bn"], p["m_tiles"], p["rounds"]) == (1, 128, 285, 5)
    p = ops.conv2d_plan(16, 19, 30, 512, 512, 3, 1)          # 72 x 4 tiles: three rounds
    assert (p["mode"], p["bn"], p["rounds"]) == (1, 128, 3)
    p = ops.conv2d_plan(16, 75, 120, 128, 128, 3, 1)         # BN = 128 on a large map: halo mode, 16 x 8 patches
    assert (p["mode"], p["bn"], p["patch_h"], p["patch_w"], p["kblocks"]) == (2, 128, 16, 8, 18)
    p = ops.conv2d_plan(16, 75, 120, 128, 128, 1, 1)         # 1x1: never halo
    assert (p["mode"], p["kblocks"], p["patch_h"], p["patch_w"]) == (1, 2, 0, 0)
    p = ops.conv2d_plan(16, 75, 120, 128, 128, 3, 1, tile_mode=1)   # linear forced: the halo layer above on linear tiles
    assert (p["mode"], p["m_tiles"], p["patch_h"], p["patch_w"]) == (1, (16 * 75 * 120 + 127) // 128, 0, 0)
    p = ops.conv2d_plan(16, 38, 60, 256, 256, 3, 1, tile_mode=2)    # halo forced: 16 x 8 patches of the 38 x 60 map
    assert (p["mode"], p["m_tiles"], p["patch_h"], p["patch_w"]) == (2, 16 * 3 * 8, 16, 8)
    p = ops.conv2d_plan(16, 38, 60, 256, 256, 3, 1, tile_mode=1, tile_bn=64)   # width forced: 4 N tiles
    assert (p["mode"], p["bn"], p["n_tiles"]) == (1, 64, 4)
    with pytest.raises(RuntimeError):
        ops.conv2d_plan(1, 8, 8, 8, 8, 5, 1)
    with pytest.raises(RuntimeError):
        ops.conv2d_plan(16, 38, 60, 256, 256, 3, 1, tile_bn=96)


def test_conv_kernels_compile_without_spills(tmp_path):
    """The tensor-core conv kernels fit their register budgets: ptxas reports 0 spill bytes for every production
    instantiation of conv_tc_kernel (TL = false) and for every conv_wgrad_kernel, and prints no warning (e.g. C7520,
    serialised wgmma) for either unit.  A spill costs speed silently; this is where a schedule change shows it first."""
    import shutil
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    procs = {src: subprocess.Popen([nvcc] + build.COMMON + ["-c", os.path.join(build.CSRC, src), "-o",
                                                            str(tmp_path / src.replace(".cu", ".o"))],
                                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for src in ("conv_tc.cu", "conv_wgrad.cu")}
    checked = []
    for src, proc in procs.items():
        out = proc.communicate(timeout=600)[0]
        assert proc.returncode == 0, out
        assert not [ln for ln in out.splitlines() if ln.startswith("ptxas") and "warning" in ln.lower()], out
        # "Compiling entry function '<mangled>'", "Function properties for <mangled>", "N bytes stack frame, S bytes spill
        # stores, L bytes spill loads"
        for name, st, ld in re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*\d+ bytes stack frame, "
                                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", out):
            if re.search(r"conv_tc_kernelILi\d+ELb0E|conv_wgrad_kernel", name):
                checked.append(name)
                assert (int(st), int(ld)) == (0, 0), f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
    assert sum("conv_tc_kernel" in n for n in checked) == 4, checked       # BN = 64 / 128 x linear / halo
    assert sum("conv_wgrad_kernel" in n for n in checked) == 3, checked    # BN = 64 / 128 / 256


def test_pack_batch_tile_table():
    """Host side of sy_pack_conv_weights_batch: items are laid out in work TILES (64 output x 32 input channels; 64 outputs of a
    stem item), `begin` is the prefix sum of sy_pack_item_tiles (a host-only entry point: no GPU needed)."""
    import torch
    from streamyolo_b200 import ops
    lib = ops.load_library()
    assert lib.sy_pack_item_tiles(64, 32, 0) == 1 and lib.sy_pack_item_tiles(65, 33, 1) == 4
    assert lib.sy_pack_item_tiles(512, 256, 0) == 8 * 8 and lib.sy_pack_item_tiles(80, 12, 2) == 2
    pb = ops.PackBatch(torch.device("cpu"))
    shapes = [((96, 80, 3, 3), 0), ((96, 80, 3, 3), 1), ((16, 12, 3, 3), 2), ((520, 264, 1, 1), 0)]
    want = 0
    for shape, mode in shapes:
        w = torch.zeros(shape)
        o, i, kh, kw = shape
        out = torch.zeros((o, kh * kw, i) if mode == 0 else ((i, kh * kw, o) if mode == 1 else (o, kh, 64)), dtype=torch.bfloat16)
        pb.add(w, out, mode, out_pitch=o if mode == 1 else 0)
        assert pb.items[-1].begin == want
        want += lib.sy_pack_item_tiles(o, i, mode)
    assert pb.total == want == 2 * 3 + 2 * 3 + 1 + 9 * 9
