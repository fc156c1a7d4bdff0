"""Generate tests/golden/contrast_script.npz -- TEST INFRASTRUCTURE.  Run in the build container, with the StreamYOLO
checkout at $STREAMYOLO_REF (default /root/reference), PIL and cv2 installed:

    python oracle/make_contrast_golden.py

The UNMODIFIED sAP/vis/vis_contrast.py main() is run under sys.argv on a fixture in a temporary directory, once per run
below, with make_videos_numbered's worker_func (imported by the script as ``make_video``) replaced by a recorder.  The
fixture is what vis_det_th.py leaves behind: two directories A and B of sequence directories of PIL-saved JPEG frames
(``Image.fromarray(rgb).save(path)``, quality 75), A and B of different content.  Sequence s0 has 18 frames of 48 x 64;
s1 has 17 frames of 37 x 53 and three of 24 x 40 among them; A's s2 has no frame, so the runs make an empty output
directory for it.  A also holds a file beside its sequences and a non-JPEG file inside s0, which the script ignores.

The runs cover the vertical and the --horizontal split, --split-pos as a fraction (0.5 of 53 is 26.5, which rounds to
26), exactly 1 (the split at the far edge: A alone, half the band) and in pixels (20), fractions that put the band
partly outside the frame (0.05, and -0.1: B alone under the band's last pixels), the swing animation at --fps 1 over
every phase (B alone, A alone, the band outside the frame) and at --fps 1.5 in between its keyframes, --seq by index
and by name, and frames skipped without --overwrite (placeholder files that the run keeps, which still advance the
animation clock) with --make-video.

Stored: the input files (in/A/..., in/B/...), and per run its extra arguments, the placeholder files made before it,
every file in its output directory afterwards, the bytes of each, what it printed to stdout (the output directory as
<out-dir>) and the recorder's calls (the video directory relative to <out-dir>, and the fps)."""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
REF = os.environ.get("STREAMYOLO_REF", "/root/reference")

from oracle.make_jpeg_encode_golden import content          # noqa: E402

SMALL = (24, 40)
SEQS = {"s0": [(48, 64)] * 18,
        "s1": [SMALL if k in (2, 9, 10) else (37, 53) for k in range(17)]}
PLACEHOLDER = b"kept"
# name -> (extra arguments, outputs made before the run)
RUNS = {
    "default": ([], []),
    "horizontal_one": (["--horizontal", "--split-pos", "1", "--overwrite"], []),
    "pixels_seq_index": (["--split-pos", "20", "--seq", "1"], []),
    "edge_seq_name": (["--split-pos", "0.05", "--seq", "s1"], []),
    "negative_horizontal": (["--split-pos", "-0.1", "--horizontal", "--seq", "s0"], []),
    "swing": (["--split-animation", "swing", "--fps", "1"], []),
    "swing_horizontal": (["--split-animation", "swing", "--fps", "1.5", "--horizontal", "--seq", "s0"], []),
    "skip_video": (["--split-animation", "swing", "--fps", "1", "--seq", "0", "--make-video"],
                   [f"s0/{k:06d}.jpg" for k in (0, 1, 2, 3, 9)]),
}


def pil_jpeg(bgr):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(bgr[..., ::-1])).save(buf, format="JPEG")
    return buf.getvalue()


def fixture():
    """{relative path under the fixture root: file bytes}"""
    files = {"A/readme.txt": b"not a sequence\n", "A/s0/thumbs.png": b"not a frame\n", "A/s2/notes.txt": b"no frames\n"}
    for s, (seq, sizes) in enumerate(SEQS.items()):
        for k, (h, w) in enumerate(sizes):
            name = f"{seq}/{k:06d}.jpg"
            files["A/" + name] = pil_jpeg(content("smooth", h, w, 1000 * s + k))
            files["B/" + name] = pil_jpeg(content("flat" if k % 3 == 0 else "smooth", h, w, 5000 + 1000 * s + k))
    return files


def import_script():
    """sAP/vis/vis_contrast.py, imported as it is"""
    sys.path.insert(0, os.path.join(REF, "sAP"))
    import vis.vis_contrast as script
    return script


def write_tree(root, files):
    for rel, b in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(b)


def run_script(script, files, extra, pre):
    """the script's main() on the fixture -> ({relative output path: bytes}, output directories, printed text, video
    calls)"""
    calls = []
    with tempfile.TemporaryDirectory() as tmp:
        write_tree(tmp, files)
        out = os.path.join(tmp, "out")
        write_tree(out, {rel: PLACEHOLDER for rel in pre})
        argv, sys.argv = sys.argv, ["vis_contrast.py", "--dir-A", os.path.join(tmp, "A"), "--dir-B",
                                    os.path.join(tmp, "B"), "--out-dir", out] + extra
        make_video, script.make_video = script.make_video, lambda args: calls.append((args[0], args[1].fps))
        printed = io.StringIO()
        try:
            with contextlib.redirect_stdout(printed), contextlib.redirect_stderr(io.StringIO()):
                script.main()
        finally:
            sys.argv = argv
            script.make_video = make_video
        written = {}
        for d, _, fs in os.walk(out):
            for f in fs:
                with open(os.path.join(d, f), "rb") as fh:
                    written[os.path.relpath(os.path.join(d, f), out)] = fh.read()
        dirs = sorted(os.path.relpath(d, out) for d, _, _ in os.walk(out) if d != out)
        videos = [(os.path.relpath(d, out), str(fps)) for d, fps in calls]
        return written, dirs, printed.getvalue().replace(out, "<out-dir>"), videos


def golden():
    script = import_script()
    files = fixture()
    g = {"runs": np.asarray(list(RUNS))}
    for rel, b in files.items():
        g["in/" + rel] = np.frombuffer(b, np.uint8)
    for run, (extra, pre) in RUNS.items():
        written, dirs, printed, videos = run_script(script, files, extra, pre)
        g[run + ".argv"] = np.asarray(extra, dtype=str)
        g[run + ".pre"] = np.asarray(pre, dtype=str)
        g[run + ".files"] = np.asarray(sorted(written), dtype=str)
        g[run + ".dirs"] = np.asarray(dirs, dtype=str)
        g[run + ".printed"] = np.asarray(printed)
        g[run + ".videos"] = np.asarray(videos, dtype=str).reshape(-1, 2)
        for rel, b in written.items():
            g[f"{run}/{rel}"] = np.frombuffer(b, np.uint8)
    return g


def main():
    path = os.path.join(ROOT, "tests", "golden", "contrast_script.npz")
    np.savez_compressed(path, **golden())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
