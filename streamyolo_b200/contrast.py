"""The sAP toolkit's method comparison (sAP/vis/vis_contrast.py) on the device: split-screen frames of two
visualisations of the same sequences, A before a split line and B after it, with an orange band at the split, written as
JPEG files byte-identical to the script's.

    python -m streamyolo_b200.contrast --dir-A vis/streamyolo --dir-B vis/baseline --out-dir vis/contrast \\
        [--horizontal] [--split-pos 0.5] [--split-animation swing] [--fps 30] [--seq 3 | --seq <name>] \\
        [--make-video] [--overwrite]

It takes the script's arguments and writes the same files: ``<out-dir>/<sequence>/<frame>`` for every ``*.jpg`` of
``<dir-A>/<sequence>``, what the script's ``Image.fromarray(img).save(path)`` writes (PIL's quality 75, which is
``cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, 75])`` byte for byte), and prints the script's lines.

The host reproduces main() (:94-175) with the script's own float64 expressions: the sorted sequence directories of
--dir-A, --seq by index or name, the output directory made even when every frame is skipped, the sorted frames, the
--overwrite skip (a skipped frame still advances the animation clock ``ii / fps``), the split position (--split-pos above
1 in pixels, otherwise a fraction of the frame's width, or height with --horizontal), the swing animation
(split_anime_swing, :45-92), ``int(round(x))`` (half to even) and the 14-pixel band [split - 7, split + 7) clamped to
the frame.  Each frame's size is read from its SOF header.  The device decodes batches of frame pairs
(data.decode_jpeg_sized, which equals PIL's decode of these files), splices them (data.splice_frames,
sy_splice_frames) and encodes at quality 75 (data.encode_jpeg); a thread pool reads and writes the files meanwhile.
--make-video runs make_videos_numbered.py's ffmpeg command once, after the loop, for the last sequence only, as the
script's indentation does; --vis-scale is accepted and unused, as in the script.

Refused:
  --split-animation other than swing   KeyError, as the script's ``globals()['split_anime_' + name]`` raises, before
                                       anything is read or written
  a frame of A without its B file      FileNotFoundError naming the B file (the script's Image.open), before the
                                       sequence's first file is written
  A and B of different sizes           ValueError naming both files (the script's numpy assignment fails on most such
                                       pairs; here on every one)
  a file the device decoder refuses    RuntimeError naming the file and the reason (data.JPEG_STATUS): not a baseline or
                                       progressive colour JPEG it reads
"""
import argparse
import errno
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import data
from .vis import _pow2, _read, _write, make_video

QUALITY = 75              # PIL's default JPEG quality, what the script's save writes with
BATCH = 8                 # frame pairs per device batch
LINE_WIDTH = 15           # the script's line_width (:105); its band is 14 pixels wide, [split - 7, split + 7)


def parse_args(argv=None):
    """vis_contrast.py's arguments (:21-36)"""
    p = argparse.ArgumentParser(prog="python -m streamyolo_b200.contrast")
    p.add_argument("--dir-A", type=str, default=None)
    p.add_argument("--dir-B", type=str, default=None)
    p.add_argument("--horizontal", action="store_true", default=False)
    p.add_argument("--split-pos", type=float, default=0.5)
    p.add_argument("--split-animation", type=str, default=None)
    p.add_argument("--fps", type=float, default=30)
    p.add_argument("--out-dir", type=str, required=True)
    p.add_argument("--vis-scale", type=float, default=1)
    p.add_argument("--seq", type=str, default=None)
    p.add_argument("--make-video", action="store_true", default=False)
    p.add_argument("--overwrite", action="store_true", default=False)
    return p.parse_args(argv)


def _ease(t):
    """the script's ease_in_out (:41-42): time in [0, 1] -> progress in [0, 1], float64"""
    return -np.cos(np.pi * t) / 2 + 0.5


def split_anime_swing(t, split_pos, l, line_width):
    """The script's swing animation (:45-92): the split held for 4 s, eased past the far edge in 1 s, held 3 s, eased
    past the near edge in 2 s, held 3 s, eased back in 1 s, then held.  Same float64 operations as the script."""
    far, near = l + line_width // 2, (-line_width) // 2 - 1
    # (seconds, start, end); end None holds start
    phases = ((4, split_pos, None), (1, split_pos, far), (3, far, None), (2, far, near), (3, near, None),
              (1, near, split_pos))
    key = 0
    for dur, start, end in phases:
        if t < key + dur:
            return start if end is None else start + _ease((t - key) / dur) * (end - start)
        key += dur
    return split_pos


ANIMATIONS = {"swing": split_anime_swing}


def frame_split(opts, ii, l):
    """Frame ``ii`` of a sequence whose frames are ``l`` pixels along the split axis -> (split, band_start, band_end) as
    sy_splice_frames takes them, clamped to [0, l]: :130-138 and the conditions of :148-165"""
    split_pos = opts.split_pos if opts.split_pos > 1 else l * opts.split_pos
    if opts.split_animation:
        split_pos = ANIMATIONS[opts.split_animation](ii / opts.fps, split_pos, l, LINE_WIDTH)
    return splice_args(int(round(split_pos)), l)


def splice_args(split, l):
    """The script's int split of a frame ``l`` pixels along the split axis -> (split, band_start, band_end) clamped to
    [0, l]: B from ``split`` on (:148-156), the band [split - 7, split + 7) where it is visible (:137-138, :158-165)"""
    start, end = split - (LINE_WIDTH - 1) // 2, split + LINE_WIDTH // 2
    if start < l and end >= 0:
        start, end = max(0, start), min(l, end)
    else:
        start = end = 0
    return min(max(split, 0), l), start, end


def sof_size(b):
    """(h, w) of a JPEG file from its SOF header, or None when there is none before the scan"""
    if b[:2] != b"\xff\xd8":
        return None
    i = 2
    while i + 4 <= len(b):
        if b[i] != 0xFF:
            return None
        m = b[i + 1]
        if m == 0xFF:                                     # fill byte
            i += 1
            continue
        if m == 0x01 or 0xD0 <= m <= 0xD7:                # no length
            i += 2
            continue
        n = (b[i + 2] << 8) | b[i + 3]
        if m in (0xC0, 0xC1, 0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF):
            if i + 9 > len(b):
                return None
            return (b[i + 5] << 8) | b[i + 6], (b[i + 7] << 8) | b[i + 8]
        if m in (0xD9, 0xDA) or n < 2:
            return None
        i += 2 + n
    return None


class Frame:
    """one output frame: its A and B files, output path and index in its sequence"""

    def __init__(self, a, b, out, ii):
        self.a, self.b, self.out, self.ii = a, b, out, ii


def pair_sizes(frames, files_a, files_b):
    """the (h, w) of each pair, from A's SOF header; ValueError where B's differs, RuntimeError without a header"""
    sizes = []
    for f, fa, fb in zip(frames, files_a, files_b):
        hw = []
        for path, b in ((f.a, fa), (f.b, fb)):
            s = sof_size(b)
            if s is None or min(s) < 1:
                raise RuntimeError(f"contrast: {path} did not decode: {data.JPEG_STATUS[1]}")
            hw.append(s)
        if hw[0] != hw[1]:
            raise ValueError(f"contrast: {f.a} is {hw[0][0]}x{hw[0][1]} but {f.b} is {hw[1][0]}x{hw[1][1]}")
        sizes.append(hw[0])
    return sizes


def device_pass(files_a, files_b, frames, opts, device="cuda"):
    """The files' bytes of a batch of Frames -> the output files: decode the 2n files, splice, encode at quality 75"""
    sizes = pair_sizes(frames, files_a, files_b)
    splits = [frame_split(opts, f.ii, h if opts.horizontal else w) for f, (h, w) in zip(frames, sizes)]
    n = len(frames)
    mh, mw = max(h for h, _ in sizes), max(w for _, w in sizes)
    files = list(files_a) + list(files_b)
    rows, lengths = data.pack_jpeg(files, _pow2(max(len(b) for b in files)))
    img, status = data.decode_jpeg_sized(torch.from_numpy(rows).to(device), torch.from_numpy(lengths).to(device),
                                         sizes + sizes, (mh, mw))
    data.splice_frames(img[:n], img[n:], splits, sizes, opts.horizontal)
    paths = [f.a for f in frames] + [f.b for f in frames]
    for p, s in zip(paths, status.tolist()):
        if s != 0:
            raise RuntimeError(f"contrast: {p} did not decode: {data.JPEG_STATUS.get(s, f'status {s}')}")
    return data.encode_jpeg(img[:n], QUALITY, sizes)


def sequence_frames(opts, seq, seq_dir_out):
    """the frames of one sequence to write (:118-126): A's sorted *.jpg files, those with an output skipped without
    --overwrite, each with its index among all of A's frames; FileNotFoundError for a missing B file"""
    seq_dir_a, seq_dir_b = os.path.join(opts.dir_A, seq), os.path.join(opts.dir_B, seq)
    names = sorted(item.name for item in os.scandir(seq_dir_a) if item.is_file() and item.name.endswith(".jpg"))
    frames = []
    for ii, name in enumerate(names):
        out = os.path.join(seq_dir_out, name)
        if not opts.overwrite and os.path.isfile(out):
            continue
        b = os.path.join(seq_dir_b, name)
        if not os.path.isfile(b):
            raise FileNotFoundError(errno.ENOENT, os.strerror(errno.ENOENT), b)
        frames.append(Frame(os.path.join(seq_dir_a, name), b, out, ii))
    return frames


def run(opts, device_pass=device_pass):
    """The script's main() with the frames composed on the device -> the number of files written; ``device_pass`` is
    the device half (tests pass an emulation)"""
    if opts.split_animation and opts.split_animation not in ANIMATIONS:
        raise KeyError("split_anime_" + opts.split_animation)
    seqs = sorted(item.name for item in os.scandir(opts.dir_A) if item.is_dir())
    if opts.seq is not None:
        idx = int(opts.seq) if opts.seq.isdigit() else seqs.index(opts.seq)
        seqs = [seqs[idx]]
    written = 0
    with ThreadPoolExecutor(max_workers=4) as pool:
        for s, seq in enumerate(seqs):
            print(f"Processing {s + 1}/{len(seqs)}: {seq}")
            seq_dir_out = os.path.join(opts.out_dir, seq)
            os.makedirs(seq_dir_out, exist_ok=True)
            frames = sequence_frames(opts, seq, seq_dir_out)
            batches = [frames[k:k + BATCH] for k in range(0, len(frames), BATCH)]
            load = lambda b: ([_read(f.a) for f in b], [_read(f.b) for f in b])     # noqa: E731
            reads = [pool.submit(load, b) for b in batches[:1]]
            writes = []
            for k, batch in enumerate(batches):
                if k + 1 < len(batches):
                    reads.append(pool.submit(load, batches[k + 1]))
                files_a, files_b = reads[k].result()
                reads[k] = None
                files = device_pass(files_a, files_b, batch, opts)
                writes += [pool.submit(_write, f.out, b) for f, b in zip(batch, files)]
            for w in writes:
                w.result()
            written += len(frames)
    if opts.make_video:
        if opts.overwrite or not os.path.isfile(seq_dir_out + ".mp4"):
            print("Making the video")
            make_video(seq_dir_out, opts.fps)
    else:
        print(f'python vis/make_videos_numbered.py "{opts.out_dir}" --fps {opts.fps}')
    return written


def main(argv=None):
    return run(parse_args(argv))


if __name__ == "__main__":
    main()
