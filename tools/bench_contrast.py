"""Split-screen comparison frames on the device (python -m streamyolo_b200.contrast, sy_splice_frames) on 1200 x 1920
frames, against the sAP toolkit's host path.

  (1) device    contrast.device_pass of n = 1, 8, 16 frame pairs after reading their 2n files from a temporary
                directory: decode of the 2n files (data.decode_jpeg_sized), splice (data.splice_frames), encode at q 75
                (data.encode_jpeg); host wall time of ``iters`` batches after warm-up (each ends in a synchronisation),
                per frame; and the splice kernel alone at n = 1 and 16 (CUDA events)
  (2) host      vis_contrast.py's per-frame work on one core: two PIL opens, the numpy splice and band, a PIL save (when
                PIL is installed; otherwise reported as not measured)
  (3) CLI       python -m streamyolo_b200.contrast on a synthetic 480-frame sequence pair with the swing animation:
                frames/s end to end

The device's files are checked against the oracle (oracle/contrast_oracle.py), encoded by the device encoder, before
anything is timed.  The card's name and power limit are read in the same run.
usage: python tools/bench_contrast.py [iters] [out path]"""
import os
import statistics
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np
import torch

from oracle import contrast_oracle as co
from oracle.make_jpeg_golden import synth_frame
from streamyolo_b200 import contrast, data

FRAME_HW = (1200, 1920)


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    out_path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(HERE), "profiles", "h100_contrast.txt")
    lines = []

    def say(s):
        print(s, flush=True)
        lines.append(s)

    try:
        from PIL import Image
    except ImportError:
        Image = None
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    say(f"$ python tools/bench_contrast.py {iters}")
    say(f"card (name, power limit, max SM clock): {card()}")
    say(f"host: {os.cpu_count()} cores, " + ("PIL" if Image else "no PIL"))
    h, w = FRAME_HW
    # inputs as vis_det_th.py leaves them: quality-75 files, A and B of different content
    host = [synth_frame(h, w, 700 + i) for i in range(32)]
    files = data.encode_jpeg(torch.from_numpy(np.stack(host)).to(dev), 75)
    with tempfile.TemporaryDirectory() as tmp:
        for side in ("A", "B"):
            os.makedirs(os.path.join(tmp, side, "s0"))
        paths_a, paths_b = [], []
        for i in range(16):
            for side, k, paths in (("A", i, paths_a), ("B", 16 + i, paths_b)):
                p = os.path.join(tmp, side, "s0", f"{i:06d}.jpg")
                open(p, "wb").write(files[k])
                paths.append(p)
        opts = contrast.parse_args(["--dir-A", os.path.join(tmp, "A"), "--dir-B", os.path.join(tmp, "B"), "--out-dir",
                                    os.path.join(tmp, "out"), "--split-animation", "swing", "--fps", "1"])
        frames = [contrast.Frame(paths_a[i], paths_b[i], "", i) for i in range(16)]
        say(f"(1) device read + decode x2 + splice + encode at q {contrast.QUALITY}, {h}x{w} frames (input files of "
            f"{statistics.mean(len(f) for f in files) / 1e3:.0f} kB; the swing's first 16 s at --fps 1)")

        def batch(n):
            fa = [contrast._read(p) for p in paths_a[:n]]
            fb = [contrast._read(p) for p in paths_b[:n]]
            return contrast.device_pass(fa, fb, frames[:n], opts)

        got = batch(16)
        rows, lengths = data.pack_jpeg(files, max(len(f) for f in files))
        dec, st = data.decode_jpeg_sized(torch.from_numpy(rows).to(dev), torch.from_numpy(lengths).to(dev),
                                         [FRAME_HW] * 32, FRAME_HW)
        assert st.cpu().eq(0).all()
        dec = dec.cpu().numpy()
        for i in range(16):                                  # against the oracle, encoded by the device encoder
            s = co.split_at(i, w, opts.split_pos, opts.split_animation, opts.fps)
            want = data.encode_jpeg(torch.from_numpy(co.compose(dec[i], dec[16 + i], s, False,
                                                                data.CONTRAST_BAND_BGR)).to(dev)[None], 75)[0]
            assert got[i] == want, i
        for n in (1, 8, 16):
            for _ in range(3):
                batch(n)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(iters):
                batch(n)
            ms = (time.perf_counter() - t0) * 1e3 / iters
            say(f"  n={n:2d}: {ms:7.2f} ms per batch (host wall, with the file reads, the copies in and out and two "
                f"synchronisations), {ms / n:6.2f} ms per frame")
        ta = torch.from_numpy(dec[:16]).to(dev)
        tb = torch.from_numpy(dec[16:]).to(dev)
        work = ta.clone()
        s_t = torch.tensor([FRAME_HW] * 16, dtype=torch.int32, device=dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for label, split in (("split at w / 2", w // 2), ("B alone", 0)):
            sp_t = torch.tensor([contrast.splice_args(split, w)] * 16, dtype=torch.int32, device=dev)
            for n in (1, 16):
                run = lambda: data.splice_frames(work[:n], tb[:n], sp_t[:n], s_t[:n])     # noqa: E731
                for _ in range(5):
                    run()
                torch.cuda.synchronize()
                a.record()
                for _ in range(iters * 5):
                    run()
                b.record()
                torch.cuda.synchronize()
                us = a.elapsed_time(b) * 1e3 / (iters * 5)
                moved = n * h * w * 3 * (2 if split == 0 else 1)          # B's bytes read and written into A
                say(f"  splice kernel alone, {label}, n={n:2d}: {us:7.1f} us per launch, {us / n:6.1f} us per frame, "
                    f"{moved / us / 1e6:.2f} TB/s of B read + A written (CUDA events)")
        if Image is not None:
            t0 = time.perf_counter()
            for i in range(8):
                img_a, img_b = Image.open(paths_a[i]), Image.open(paths_b[i])
                img = np.array(img_a)
                img_b = np.asarray(img_b)
                img[:, w // 2:] = img_b[:, w // 2:]
                img[:, w // 2 - 7:w // 2 + 7] = np.array([241, 159, 93], np.uint8).reshape(1, 1, 3)
                Image.fromarray(img).save(os.path.join(tmp, f"host{i}.jpg"))
            ms = (time.perf_counter() - t0) * 1e3 / 8
            say(f"(2) host path: {ms:.1f} ms per frame on one core (two PIL opens, numpy splice, PIL save)")
        else:
            say("(2) host path: not measured (no PIL on this host)")
        n_frames = 480
        for side, off in (("A", 0), ("B", 16)):
            os.makedirs(os.path.join(tmp, "cli", side, "s0"))
            for i in range(n_frames):
                open(os.path.join(tmp, "cli", side, "s0", f"{i:06d}.jpg"), "wb").write(files[off + i % 16])
        argv = ["--dir-A", os.path.join(tmp, "cli", "A"), "--dir-B", os.path.join(tmp, "cli", "B"), "--out-dir",
                os.path.join(tmp, "cli", "out"), "--split-animation", "swing", "--overwrite"]
        walls = []
        with open(os.devnull, "w") as nul:
            old, sys.stdout = sys.stdout, nul
            try:
                for _ in range(3):                           # the first is the warm-up
                    t0 = time.perf_counter()
                    contrast.run(contrast.parse_args(argv))
                    walls.append(time.perf_counter() - t0)
            finally:
                sys.stdout = old
        wall = min(walls[1:])
        say(f"(3) CLI, {n_frames} frame pairs of {h}x{w}, swing at 30 fps: {wall:.2f} s, {n_frames / wall:.0f} frames/s "
            f"(best of {len(walls) - 1})")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
