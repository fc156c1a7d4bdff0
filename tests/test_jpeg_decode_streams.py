"""Device JPEG decode (streamyolo_b200.data.decode_jpeg / decode_jpeg_sized) against its numpy oracle on generated and
adversarial streams.

Four families of streams:
  fixture     tests/golden/jpeg_streams.npz (oracle/make_jpeg_streams_golden.py): cv2-written 4:2:2 and 4:4:4 files,
              optimised tables, restart intervals of 1 (36 000 of them in a 1200 x 1920 frame), of a count that does not
              divide the MCUs and of more than the MCUs, q100 noise; with cv2's pixels or their hashes
  generated   4:2:0 files of oracle/jpeg_encode_oracle.py (byte-identical to cv2.imencode) at seeded sizes from 1 x 1 to
              1200 x 1920, qualities 1 .. 100 and every content kind of make_jpeg_encode_golden.content; a 1200 x 1920
              q100 noise frame holds more than 1 MiB of entropy-coded data
  crafted     quantised coefficients written straight into a scan: every AC zero (periodic bitstreams), repeated tiles,
              a coefficient at index 63 (no EOB), ZRL chains, DC differences alternating at category 11, Huffman tables of
              16-bit codes, scans of 1, 2 and exactly 4096 subsequences, 1-bits after the last block, and restart streams
              with more than 4096 intervals
  rewritten   byte-level rewrites of cv2's files that leave the pixels alone: COM / APPn segments, 16-bit DQT, merged
              table segments, renumbered tables, component ids 0 / 1 / 2, DRI 0, fill bytes before markers, bytes after EOI

CPU: the oracle equals cv2.imdecode on every family (the generated 1200 x 1920 frame excepted: it is too slow for the
     oracle, and its encoder is pinned to cv2 in test_jpeg_encode.py) and the fixture's hashes; every rewrite decodes in
     cv2 as its original does; the streams reach the decoder's paths (subsequence counts of 1, 2 and 4096, a subsequence
     longer than 2048 bits, a scan of a whole number of subsequences, more than 4096 restart intervals, every sampling at
     MCU-aligned and unaligned sizes).
GPU: decode_jpeg and decode_jpeg_sized equal the oracle (or cv2's hashes) on every stream in batches of mixed sizes, and
     one decode_jpeg_sized launch of every sampling, restart and self-synchronising streams, a 1 x 1 frame, a frame of the
     slot's size and a damaged stream writes no pixel outside each image.
"""
import functools
import hashlib
import os
import re

import numpy as np
import pytest
import torch

from oracle import jpeg_encode_oracle as je
from oracle import jpeg_oracle as jo
from oracle import make_jpeg_streams_golden as mks
from oracle.make_jpeg_encode_golden import CONTENTS, content
from oracle.make_jpeg_golden import exif_app1
from streamyolo_b200 import data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = dict(np.load(os.path.join(ROOT, "tests", "golden", "jpeg_streams.npz")))
FIX_NAMES = sorted(mks.CASES)

SAMP = {"420": (2, 2), "422": (2, 1), "444": (1, 1)}
MAX_SUBSEQ, MIN_SUBSEQ_BITS = 4096, 2048       # jpeg.cu kMaxSubseq, kMinSubseqBits


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------ stream families
# generated: (h, w, quality, content); edge sizes first (1 x N, N x 1, w <= 4 where the chroma plane is at most 2 samples
# wide, MCU-aligned), then seeded random sizes, a 600 x 960 frame and the 1200 x 1920 q100 noise frame
def _generated_cases():
    edge = [(1, 1, 1, "smooth"), (1, 57, 37, "noise"), (61, 1, 64, "checker"), (2, 2, 100, "noise"), (3, 4, 88, "flat"),
            (4, 3, 13, "checker"), (7, 2, 50, "smooth"), (9, 4, 97, "noise"), (16, 32, 75, "smooth"),
            (48, 64, 100, "noise"), (32, 16, 5, "flat"), (240, 320, 100, "noise")]
    r = np.random.default_rng(2024)
    rand = []
    for k in range(10):
        h, w = int(r.integers(1, 300)), int(r.integers(1, 500))
        rand.append((h, w, int(r.integers(1, 101)), CONTENTS[k % len(CONTENTS)]))
    return edge + rand + [(600, 960, int(r.integers(1, 101)), "smooth"), (1200, 1920, 100, "noise")]


GENERATED = {f"g{h}x{w}_q{q}_{kind}": (h, w, q, kind) for h, w, q, kind in _generated_cases()}
SLOW_GENERATED = {"g1200x1920_q100_noise"}      # not decoded by the oracle on the CPU


@functools.lru_cache(maxsize=None)
def generated(name):
    h, w, q, kind = GENERATED[name]
    return je.encode(content(kind, h, w, sorted(GENERATED).index(name)), q)


# --- header segments
def _segments(b):
    """a file's header as [marker, payload] pairs from after SOI through SOS, and the bytes after SOS"""
    segs, i = [], 2
    while True:
        while b[i] == 0xFF and b[i + 1] == 0xFF:
            i += 1
        m, ln = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        segs.append([m, bytes(b[i + 4:i + 2 + ln])])
        i += 2 + ln
        if m == 0xDA:
            return segs, bytes(b[i:])


def _join(segs, rest, fill=b""):
    """the file of ``segs`` and ``rest``, with ``fill`` before every marker after SOI"""
    return b"\xff\xd8" + b"".join(fill + bytes([0xFF, m]) + (len(p) + 2).to_bytes(2, "big") + p for m, p in segs) + rest


def _dht(tc, th, counts, symbols):
    return bytes([(tc << 4) | th]) + bytes(counts) + bytes(symbols)


# --- crafted scans
def _codes(counts, symbols):
    return {s: format(c, f"0{ln}b") for s, (c, ln) in je.huff_codes(counts, symbols).items()}


STD_CODES = [(_codes(*je.STD_HUFF["dc0"]), _codes(*je.STD_HUFF["ac0"])),
             (_codes(*je.STD_HUFF["dc1"]), _codes(*je.STD_HUFF["ac1"]))]


def _extra(v, s):
    return format((v if v >= 0 else v - 1) & ((1 << s) - 1), f"0{s}b") if s else ""


def _block(row, prev, dc, ac):
    """the bits of one block of zigzag coefficients ``row`` after a block of DC ``prev`` (jchuff.c encode_one_block)"""
    diff = int(row[0]) - prev
    s = abs(diff).bit_length()
    out = [dc[s], _extra(diff, s)]
    last = 0
    for k in np.flatnonzero(row[1:]) + 1:
        run = int(k) - last - 1
        while run > 15:
            out.append(ac[0xF0])
            run -= 16
        v = int(row[k])
        s = abs(v).bit_length()
        out += [ac[(run << 4) | s], _extra(v, s)]
        last = int(k)
    if last < 63:
        out.append(ac[0x00])
    return "".join(out)


def _scan(coef, samp, ri=0, codes=None):
    """the byte-stuffed entropy-coded segment of zigzag coefficients [mcus * blocks per MCU, 64] in MCU order: DC
    predictions reset and an RSTn marker written every ``ri`` MCUs, each interval padded with 1-bits"""
    h0, v0 = SAMP[samp]
    comp_of = [0] * (h0 * v0) + [1, 2]
    bpm = len(comp_of)
    codes = codes or [STD_CODES[0], STD_CODES[1], STD_CODES[1]]
    mcus = coef.shape[0] // bpm
    per = ri or mcus
    out = bytearray()
    for k, m0 in enumerate(range(0, mcus, per)):
        if k:
            out += bytes([0xFF, 0xD0 + (k - 1) % 8])
        pred, bits = [0, 0, 0], []
        for b in range(m0 * bpm, min(m0 + per, mcus) * bpm):
            c = comp_of[b % bpm]
            bits.append(_block(coef[b], pred[c], *codes[c]))
            pred[c] = int(coef[b, 0])
        s = "".join(bits)
        s += "1" * (-len(s) % 8)
        out += je.stuff(np.packbits(np.frombuffer(s.encode(), np.uint8) - 48).tobytes())
    return bytes(out)


def _file(h, w, q, samp, scan, ri=0, dht=None):
    """je.header's segments with the sampling ``samp``, a DRI of ``ri`` when nonzero and the DHT payloads ``dht`` (the
    standard tables when None), then ``scan`` and EOI"""
    segs, _ = _segments(je.header(h, w, q))
    h0, v0 = SAMP[samp]
    out = []
    for m, p in segs:
        if m == 0xC0:
            p = p[:7] + bytes([(h0 << 4) | v0]) + p[8:]
        if m == 0xC4:
            if dht is None:
                out.append([m, p])
            elif dht:
                out += [[0xC4, d] for d in dht]
                dht = []
            continue
        if m == 0xDA and ri:
            out.append([0xDD, ri.to_bytes(2, "big")])
        out.append([m, p])
    return _join(out, scan + b"\xff\xd9")


def _mcus(h, w, samp):
    h0, v0 = SAMP[samp]
    return _cdiv(h, 8 * v0) * _cdiv(w, 8 * h0), h0 * v0 + 2


def _random_coef(r, n, density, max_cat, dc_step=8):
    """n blocks of zigzag coefficients: AC nonzero with probability ``density``, of categories 1 .. max_cat, and a DC
    random walk"""
    coef = np.zeros((n, 64), np.int64)
    cat = r.integers(1, max_cat + 1, (n, 63))
    mag = (1 << (cat - 1)) + (r.integers(0, 1 << 20, (n, 63)) & ((1 << (cat - 1)) - 1))
    coef[:, 1:] = np.where(r.random((n, 63)) < density, mag * r.choice([-1, 1], (n, 63)), 0)
    coef[:, 0] = np.clip(np.cumsum(r.integers(-dc_step, dc_step + 1, n)), -1000, 1000)
    return coef


def _tame(coef, samp, q, budget=1000):
    """coefficients an 8-bit image could have: each block's dequantised DC within +-1024 and the L1 norm of its
    dequantised AC within ``budget``, so that every IDCT sample stays inside libjpeg's range-limit table and the 16-bit
    intermediates of libjpeg-turbo's SIMD IDCT, where the C and SIMD IDCTs agree"""
    h0, v0 = SAMP[samp]
    qt = je.quant_tables(q)[:, jo.ZIGZAG]
    comp = np.tile([0] * (h0 * v0) + [1, 1], coef.shape[0] // (h0 * v0 + 2))
    dq = qt[comp]
    coef = coef.copy()
    coef[:, 0] = np.clip(coef[:, 0], -(1024 // dq[:, 0]), 1024 // dq[:, 0] - (dq[:, 0] == 1))
    l1 = (np.abs(coef[:, 1:]) * dq[:, 1:]).sum(axis=1, keepdims=True)
    scaled = np.sign(coef[:, 1:]) * np.maximum(np.abs(coef[:, 1:]) * budget // np.maximum(l1, 1), 1)
    coef[:, 1:] = np.where((l1 > budget) & (coef[:, 1:] != 0), scaled, coef[:, 1:])
    assert ((np.abs(coef[:, 1:]) * dq[:, 1:]).sum(axis=1) <= budget + 64 * dq[:, 1:].max(axis=1)).all()
    return coef


def _exact_units(r):
    """a 4:2:0 q100 scan of exactly 4096 x 2048 bits (destuffed): 4096 subsequences of 2048 bits, the last ending at the
    scan's end.  Dense random MCUs, then MCUs of zero DC difference whose luma blocks carry runs of +1 coefficients (3 bits
    each) to make up the rest"""
    h, w = 896, 896
    mcus, bpm = _mcus(h, w, "420")
    target = MAX_SUBSEQ * MIN_SUBSEQ_BITS
    coef = _tame(_random_coef(r, mcus * bpm, 1.0, 6), "420", 100, budget=1400)
    comp_of = [0, 0, 0, 0, 1, 2]
    cost, pred = np.zeros(mcus, np.int64), [0, 0, 0]
    for b in range(mcus * bpm):
        c = comp_of[b % bpm]
        cost[b // bpm] += len(_block(coef[b], pred[c], *STD_CODES[min(c, 1)]))
        pred[c] = int(coef[b, 0])
    cum = np.concatenate([[0], np.cumsum(cost)])
    for bulk in range(mcus, 0, -1):            # dense MCUs, then tail MCUs of 32 bits plus up to 4 * 62 * 3
        rest = target - cum[bulk] - 32 * (mcus - bulk)
        if 0 <= rest <= 4 * 62 * 3 * (mcus - bulk):
            break
    last_dc = coef[bulk * bpm - 3:bulk * bpm, 0]    # the last luma, Cb and Cr DC before the tail
    coef[bulk * bpm:] = 0
    coef[bulk * bpm:, 0] = np.tile(last_dc[[0, 0, 0, 0, 1, 2]], mcus - bulk)
    ones = rest // 3
    for b in range(bulk * bpm, mcus * bpm):
        if ones == 0:
            break
        if comp_of[b % bpm] == 0:
            k = min(ones, 62)
            coef[b, 1:k + 1] = 1
            ones -= k
    return _file(h, w, 100, "420", _scan(coef, "420"))


def _long_code_tables():
    """DHT payloads whose codes run to 16 bits: DC categories at lengths 2 .. 12 and 16; AC symbols at lengths 2 .. 16
    and the rest at 16 bits, the EOB and the common symbols among the longest"""
    dc_counts = [0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1]
    ac_syms = [0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11) if (r, s) != (0, 1) and (r, s) != (0, 2)]
    ac_syms = ac_syms[:14] + [0x01, 0x02, 0x00] + ac_syms[14:]
    ac_counts = [0] + [1] * 14 + [len(ac_syms) - 14]
    tabs = [(dc_counts, list(range(12))), (ac_counts, ac_syms)]
    payloads = [_dht(tc, th, *tabs[tc]) for th in (0, 1) for tc in (0, 1)]
    codes = (_codes(*tabs[0]), _codes(*tabs[1]))
    return payloads, codes


def _crafted_bytes(name):
    r = np.random.default_rng(sorted(CRAFTED).index(name) + 77)
    if name == "flat_ac0_1200x1920":           # every block the same: a stream of one 32-bit period
        mcus, bpm = _mcus(1200, 1920, "420")
        coef = np.zeros((mcus * bpm, 64), np.int64)
        coef[:, 0] = 12
        return _file(1200, 1920, 75, "420", _scan(coef, "420"))
    if name == "tiles_600x960":                # one 4:2:0 MCU of sparse coefficients repeated
        mcus, bpm = _mcus(600, 960, "420")
        tile = _tame(_random_coef(r, bpm, 0.3, 5), "420", 85)
        return _file(600, 960, 85, "420", _scan(np.tile(tile, (mcus, 1)), "420"))
    if name == "ac0_dcwalk_444_200x328":       # every AC zero, the DC wandering (4:4:4)
        mcus, bpm = _mcus(200, 328, "444")
        coef = np.zeros((mcus * bpm, 64), np.int64)
        coef[:, 0] = np.cumsum(r.integers(-3, 4, mcus * bpm))
        return _file(200, 328, 90, "444", _scan(coef, "444"))
    if name == "no_eob_240x320":               # index 63 nonzero in every block: no EOB anywhere
        mcus, bpm = _mcus(240, 320, "420")
        coef = _random_coef(r, mcus * bpm, 0.2, 6)
        coef[:, 63] = r.choice([-3, -1, 1, 2], mcus * bpm)
        coef = _tame(coef, "420", 95)
        return _file(240, 320, 95, "420", _scan(coef, "420"))
    if name == "zrl_chains_422_120x200":       # one to three ZRLs before each of a few coefficients
        mcus, bpm = _mcus(120, 200, "422")
        coef = np.zeros((mcus * bpm, 64), np.int64)
        coef[:, 0] = np.cumsum(r.integers(-5, 6, mcus * bpm))
        for b in range(mcus * bpm):
            k = int(r.choice([16, 17, 32, 33, 48, 49, 63]))
            coef[b, k] = r.choice([-7, 1, 5])
            if k < 40 and r.random() < 0.5:
                coef[b, 63] = 2
        return _file(120, 200, 80, "422", _scan(coef, "422"))
    if name == "dc_cat11_160x240":             # DC differences of +-2047 in every component
        mcus, bpm = _mcus(160, 240, "420")
        coef = _tame(_random_coef(r, mcus * bpm, 0.1, 4), "420", 100)
        comp_of = np.tile([0, 0, 0, 0, 1, 2], mcus)
        seq = np.zeros(mcus * bpm, np.int64)
        for c in range(3):
            idx = np.flatnonzero(comp_of == c)
            seq[idx] = np.where(np.arange(idx.size) & 1, 1023, -1024)
        coef[:, 0] = seq
        return _file(160, 240, 100, "420", _scan(coef, "420"))
    if name == "long_codes_176x256":           # every code 9 .. 16 bits except a few
        payloads, codes = _long_code_tables()
        mcus, bpm = _mcus(176, 256, "420")
        coef = _tame(_random_coef(r, mcus * bpm, 0.25, 10), "420", 90)
        return _file(176, 256, 90, "420", _scan(coef, "420", codes=[codes] * 3), dht=payloads)
    if name == "units_4096_exact_896x896":
        return _exact_units(r)
    if name == "units_2_16x32":                # 2048 < bits <= 4096
        mcus, bpm = _mcus(16, 32, "420")
        return _file(16, 32, 100, "420", _scan(_tame(_random_coef(r, mcus * bpm, 0.5, 4), "420", 100), "420"))
    if name == "units_1_8x8":
        return _file(8, 8, 60, "420", _scan(_tame(_random_coef(r, 6, 0.3, 3), "420", 60), "420"))
    if name == "tail_ones_96x128":             # 2400 1-bits (stuffed FF bytes) after the last block
        mcus, bpm = _mcus(96, 128, "420")
        f = _file(96, 128, 90, "420", _scan(_tame(_random_coef(r, mcus * bpm, 0.6, 6), "420", 90), "420"))
        return f[:-2] + b"\xff\x00" * 300 + b"\xff\xd9"
    if name == "rst_ri1_ac0_1200x1920":        # 9000 restart intervals of one MCU each
        mcus, bpm = _mcus(1200, 1920, "420")
        coef = np.zeros((mcus * bpm, 64), np.int64)
        coef[:, 0] = r.integers(-60, 61, mcus * bpm)
        coef[::7, 1] = 3
        return _file(1200, 1920, 75, "420", _scan(coef, "420", 1), ri=1)
    if name == "rst_ri7_422_96x136":           # dense content, 7 not dividing the 108 MCUs
        mcus, bpm = _mcus(96, 136, "422")
        return _file(96, 136, 100, "422", _scan(_tame(_random_coef(r, mcus * bpm, 0.7, 9), "422", 100), "422", 7), ri=7)
    raise KeyError(name)


CRAFTED = ["flat_ac0_1200x1920", "tiles_600x960", "ac0_dcwalk_444_200x328", "no_eob_240x320", "zrl_chains_422_120x200",
           "dc_cat11_160x240", "long_codes_176x256", "units_4096_exact_896x896", "units_2_16x32", "units_1_8x8",
           "tail_ones_96x128", "rst_ri1_ac0_1200x1920", "rst_ri7_422_96x136"]


@functools.lru_cache(maxsize=None)
def crafted(name):
    return _crafted_bytes(name)


# --- rewrites of cv2's files
def _dqt16(segs):
    out = []
    for m, p in segs:
        if m == 0xDB:
            q = b""
            for o in range(0, len(p), 65):
                q += bytes([0x10 | p[o]]) + np.frombuffer(p[o + 1:o + 65], np.uint8).astype(">u2").tobytes()
            p = q
        out.append([m, p])
    return out


def _merged(segs):
    """all DQT tables in one segment and all DHT tables (AC first) in another, where the first of each stood"""
    dqt = b"".join(p for m, p in segs if m == 0xDB)
    dht = b"".join(p for m, p in segs if m == 0xC4 and p[0] >> 4 == 1) + b"".join(
        p for m, p in segs if m == 0xC4 and p[0] >> 4 == 0)
    out, seen = [], set()
    for m, p in segs:
        if m in (0xDB, 0xC4):
            if m not in seen:
                out.append([m, dqt if m == 0xDB else dht])
                seen.add(m)
            continue
        out.append([m, p])
    return out


def _renumbered(segs, qmap, hmap_dc, hmap_ac, cr=None):
    """table ids through the maps in DQT, DHT, SOF and SOS; ``cr`` (quant id, DC id, AC id) gives Cr copies of its tables
    under those ids"""
    out = []
    for m, p in segs:
        p = bytearray(p)
        if m == 0xDB:
            extra = b""
            for o in range(0, len(p), 65):
                tq = p[o] & 15
                if cr and tq == 1:
                    extra += bytes([cr[0]]) + bytes(p[o + 1:o + 65])
                p[o] = (p[o] & 0xF0) | qmap[tq]
            p += extra
        elif m == 0xC4:
            tc, th = p[0] >> 4, p[0] & 15
            if cr and th == 1:
                out.append([m, bytes([(tc << 4) | cr[1 + tc]]) + bytes(p[1:])])
            p[0] = (tc << 4) | (hmap_ac if tc else hmap_dc)[th]
        elif m == 0xC0:
            for k in range(3):
                p[8 + 3 * k] = qmap[p[8 + 3 * k]]
            if cr:
                p[14] = cr[0]
        elif m == 0xDA:
            for k in range(3):
                t = p[2 + 2 * k]
                p[2 + 2 * k] = (hmap_dc[t >> 4] << 4) | hmap_ac[t & 15]
            if cr:
                p[6] = (cr[1] << 4) | cr[2]
        out.append([m, bytes(p)])
    return out


def _component_ids(segs, ids):
    out = []
    for m, p in segs:
        p = bytearray(p)
        if m == 0xC0:
            for k in range(3):
                p[6 + 3 * k] = ids[k]
        elif m == 0xDA:
            for k in range(3):
                p[1 + 2 * k] = ids[k]
        out.append([m, bytes(p)])
    return out


def _insert_before(segs, marker, new):
    k = next(i for i, (m, _) in enumerate(segs) if m == marker)
    return segs[:k] + new + segs[k:]


COM = [0xFE, b"written by a camera \xff\xd8 not a marker"]
APPS = [[0xE1, exif_app1(1)[4:]], [0xE2, b"ICC_PROFILE\x00" + bytes(range(40))], [0xED, b"Photoshop 3.0\x00"],
        [0xEF, b""]]

REWRITES = {
    "com_app": lambda s, r: (_insert_before(s, 0xDB, APPS + [COM]), r),
    "com_before_sos": lambda s, r: (_insert_before(s, 0xDA, [COM, COM]), r),
    "dqt16": lambda s, r: (_dqt16(s), r),
    "tables_merged": lambda s, r: (_merged(s), r),
    "tables_merged_dqt16": lambda s, r: (_merged(_dqt16(s)), r),
    "table_ids_swapped": lambda s, r: (_renumbered(s, [1, 0, 2, 3], [1, 0, 2, 3], [1, 0, 2, 3]), r),
    "table_ids_cr_own": lambda s, r: (_renumbered(s, [3, 0, 2, 1], [2, 3, 0, 1], [1, 2, 3, 0], cr=(2, 1, 0)), r),
    "component_ids_012": lambda s, r: (_component_ids(s, [0, 1, 2]), r),
    "dri0": lambda s, r: (_insert_before(s, 0xDA, [[0xDD, b"\x00\x00"]]), r),
    "fill_before_markers": lambda s, r: (s, re.sub(rb"\xff[\xd0-\xd7\xd9]", lambda m: b"\xff\xff" + m.group(0), r)),
    "after_eoi": lambda s, r: (s, r + b"\x00\x11\xff\xd8\xff\xe0 trailing bytes\xff"),
}
FILLED = {"fill_before_markers"}                # also writes fill bytes before the header's markers
REWRITE_BASES = ["s420_q90_31x47", "s420_q85_r1000_33x65", "s422_q90_opt_r7_45x77", "s444_q95_r1_37x53"]


@functools.lru_cache(maxsize=None)
def rewritten(name):
    kind, base = name.split("@")
    segs, rest = _segments(FIX[base + ".jpg"].tobytes())
    segs, rest = REWRITES[kind]([list(x) for x in segs], rest)
    return _join(segs, rest, b"\xff\xff" if kind in FILLED else b"")


REWRITTEN = [f"{k}@{b}" for k in REWRITES for b in REWRITE_BASES if not (k == "dri0" and "_r" in b)]

FAMILIES = {"generated": (sorted(GENERATED), generated), "crafted": (CRAFTED, crafted),
            "rewritten": (REWRITTEN, rewritten)}


# ------------------------------------------------------------------------------------------------------ helpers
def _hw(b):
    hd = jo.parse(b)
    return hd["h"], hd["w"]


def _band(b):
    return 8 * jo.parse(b)["comps"][0][2]


def _first_bad_row(name, got, want, band):
    """equal, or an assertion naming the first MCU row that differs"""
    if np.array_equal(got, want):
        return
    rows = np.nonzero((got != want).reshape(got.shape[0], -1).any(axis=1))[0]
    r = int(rows[0]) // band
    raise AssertionError(f"{name}: first wrong MCU row {r} (pixel rows {r * band}..), {rows.size} pixel rows differ")


def _check_fixture(name, img):
    if name + ".bgr" in FIX:
        return _first_bad_row(name, img, FIX[name + ".bgr"], mks.band(mks.CASES[name][3]))
    want = FIX[name + ".rows"]
    got = mks.row_crcs(img, mks.CASES[name][3])
    bad = np.nonzero(got != want)[0]
    band = mks.band(mks.CASES[name][3])
    assert bad.size == 0, f"{name}: first wrong MCU row {bad[0]} (pixel rows {bad[0] * band}..)"
    assert hashlib.sha256(np.ascontiguousarray(img).tobytes()).digest() == FIX[name + ".sha256"].tobytes(), name


@functools.lru_cache(maxsize=None)
def _oracle(family, name):
    b = FAMILIES[family][1](name)
    img, st = jo.decode(b)
    assert st == jo.OK, (name, jo.STATUS_NAMES[st])
    return img


def _units(b):
    """(sampling, h, w, restart intervals, n_units, unit_bits, ecs bits) as jpeg_ecs_kernel sets them"""
    hd = jo.parse(b)
    segs = jo.split_scan(bytes(b), hd["scan"])
    samp = {v: k for k, v in SAMP.items()}[hd["comps"][0][1:3]]
    bits = 8 * sum(len(s) for s in segs)
    if hd["ri"]:
        return samp, hd["h"], hd["w"], len(segs), len(segs), 0, bits
    ub = max(MIN_SUBSEQ_BITS, _cdiv(_cdiv(bits, MAX_SUBSEQ), 32) * 32)
    return samp, hd["h"], hd["w"], 0, max(1, _cdiv(bits, ub)), ub, bits


def _all_streams():
    out = {("fixture", n): FIX[n + ".jpg"].tobytes() for n in FIX_NAMES}
    for fam, (names, fn) in FAMILIES.items():
        out.update({(fam, n): fn(n) for n in names})
    return out


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_fixture_version_and_oracle():
    assert "libjpeg-turbo" in str(FIX["libjpeg_turbo"])
    for name in FIX_NAMES:
        img, st = jo.decode(FIX[name + ".jpg"])
        assert st == jo.OK, name
        _check_fixture(name, img)


def test_fixture_reproduces():
    """make_jpeg_streams_golden writes the same files with this cv2"""
    cv2 = pytest.importorskip("cv2")
    from oracle.make_jpeg_encode_golden import libjpeg_turbo_version
    if libjpeg_turbo_version() != str(FIX["libjpeg_turbo"]):
        pytest.skip("another libjpeg-turbo than the fixture's")
    for name in FIX_NAMES:
        b = mks.case_bytes(name)
        assert b == FIX[name + ".jpg"].tobytes(), name
        _check_fixture(name, cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR))


@pytest.mark.parametrize("family,name", [("generated", n) for n in sorted(GENERATED) if n not in SLOW_GENERATED] +
                         [("crafted", n) for n in CRAFTED] + [("rewritten", n) for n in REWRITTEN])
def test_oracle_equals_cv2(family, name):
    cv2 = pytest.importorskip("cv2")
    b = FAMILIES[family][1](name)
    want = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    assert want is not None and want.shape[:2] == _hw(b)
    _first_bad_row(name, _oracle(family, name), want, _band(b))
    if family == "rewritten":                   # the rewrite leaves cv2's pixels alone
        assert np.array_equal(want, FIX[name.split("@")[1] + ".bgr"]), name


def test_rewrites_change_the_bytes_only_as_named():
    for name in REWRITTEN:
        b, base = rewritten(name), FIX[name.split("@")[1] + ".jpg"].tobytes()
        assert b != base, name
        hd, hb = jo.parse(b), jo.parse(base)
        assert (hd["h"], hd["w"], [c[1:3] for c in hd["comps"]]) == (hb["h"], hb["w"], [c[1:3] for c in hb["comps"]])
        assert all(np.array_equal(a, c) for a, c in zip(hd["q"], hb["q"])), name
        if name.startswith("dqt16"):
            assert all(p[0] >> 4 == 1 for m, p in _segments(b)[0] if m == 0xDB)
        if name.startswith("component_ids"):
            assert [c[0] for c in hd["comps"]] == [0, 1, 2]
        if name.startswith("dri0"):
            assert hd["ri"] == 0


def test_streams_reach_every_decoder_path():
    """the suite's streams reach the paths of jpeg_ecs_kernel / jpeg_huffman_kernel: subsequence counts of 1, 2 and 4096
    (kMaxSubseq), a subsequence longer than 2048 bits (a scan above 1 MiB), a scan of a whole number of subsequences,
    more than 4096 restart intervals (the strided interval loop), and every sampling at MCU-aligned and unaligned sizes"""
    info = {k: _units(b) for k, b in _all_streams().items()}
    selfsync = [v for v in info.values() if v[3] == 0]
    counts = {v[4] for v in selfsync}
    assert {1, 2, MAX_SUBSEQ} <= counts, sorted(counts)
    assert any(v[5] > MIN_SUBSEQ_BITS for v in selfsync)
    assert any(v[6] == v[4] * v[5] and v[4] > 1 for v in selfsync)
    assert max(v[3] for v in info.values()) > MAX_SUBSEQ
    assert any(v[3] > MAX_SUBSEQ for k, v in info.items() if k[0] == "fixture")
    assert max(len(generated(n)) for n in GENERATED) > (1 << 20) + je.HEADER_BYTES
    for samp, (h0, v0) in SAMP.items():
        aligned = {v[1] % (8 * v0) == 0 and v[2] % (8 * h0) == 0 for v in info.values() if v[0] == samp}
        assert aligned == {True, False}, samp
    # the crafted edges: 16-bit codes, no EOB, category-11 DC differences, ZRLs
    hd = jo.parse(crafted("long_codes_176x256"))
    assert max(ln for ln, _ in hd["huff"][0][1]) == 16


def test_crafted_scans_hold_their_edges():
    """each crafted scan decodes (oracle) to the coefficients it was built for: index 63 set in every no-EOB block, DC
    differences of 2047, ZRL runs, a 2-subsequence and a 1-subsequence scan, the 1-bit tail"""
    assert _units(crafted("units_2_16x32"))[4] == 2
    assert _units(crafted("units_1_8x8"))[4] == 1
    u = _units(crafted("units_4096_exact_896x896"))
    assert u[4:] == (MAX_SUBSEQ, MIN_SUBSEQ_BITS, MAX_SUBSEQ * MIN_SUBSEQ_BITS)
    u = _units(crafted("tail_ones_96x128"))
    b = crafted("tail_ones_96x128")
    hd = jo.parse(b)
    seg = jo.split_scan(b, hd["scan"])[0]
    assert seg.endswith(b"\xff" * 300) and u[4] >= 3
    for name in ("no_eob_240x320", "dc_cat11_160x240", "zrl_chains_422_120x200"):
        b = crafted(name)
        hd = jo.parse(b)
        coef, _ = jo.entropy_decode(hd, jo.split_scan(b, hd["scan"]))
        if name.startswith("no_eob"):
            assert (coef[:, 63] != 0).all()
        elif name.startswith("dc_cat11"):
            comp = np.tile([0, 0, 0, 0, 1, 2], coef.shape[0] // 6)
            for c in range(3):
                d = np.diff(coef[comp == c, 0])
                assert (np.abs(d) == 2047).all()
        else:
            nz = coef != 0
            assert nz[:, 1:].any(axis=1).all() and nz[:, jo.ZIGZAG[1:16]].sum() == 0


# ---------------------------------------------------------------------------------------------------------------- GPU
SENTINEL = 0xA5


def _pack(files):
    rows, lengths = data.pack_jpeg([np.frombuffer(f, np.uint8) for f in files], max(len(f) for f in files) + 64)
    return torch.from_numpy(rows).cuda(), torch.from_numpy(lengths).cuda()


def _decode_sized_checked(files, sizes, max_hw):
    """decode_jpeg_sized into slots pre-filled with SENTINEL: -> host frames and statuses, asserting that no pixel
    outside an image (or of a refused image) changed"""
    s, l = _pack(files)
    out = torch.full((len(files), *max_hw, 3), SENTINEL, dtype=torch.uint8, device="cuda")
    frames, status = data.decode_jpeg_sized(s, l, sizes, max_hw, out=out)
    st = status.cpu().tolist()
    f = frames.cpu().numpy()
    for k, (h, w) in enumerate(sizes):
        m = np.ones(max_hw, bool)
        if st[k] == 0:
            m[:h, :w] = False
        assert (f[k][m] == SENTINEL).all(), f"frame {k} ({h}x{w}, status {st[k]}): pixels outside the image written"
    return f, st


def _batches(names, fn, max_bytes=24 << 20):
    """names in batches of mixed sizes whose files together stay under max_bytes"""
    out, cur, tot = [], [], 0
    for n in sorted(names, key=lambda n: len(fn(n))):
        if cur and tot + len(fn(n)) > max_bytes:
            out.append(cur)
            cur, tot = [], 0
        cur.append(n)
        tot += len(fn(n))
    return out + [cur]


@pytest.mark.gpu
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_gpu_streams_equal_oracle(family):
    names, fn = FAMILIES[family]
    for batch in _batches(names, fn):
        files = [fn(n) for n in batch]
        sizes = [_hw(b) for b in files]
        max_hw = (max(h for h, _ in sizes), max(w for _, w in sizes))
        frames, st = _decode_sized_checked(files, sizes, max_hw)
        for k, n in enumerate(batch):
            assert st[k] == 0, (n, jo.STATUS_NAMES.get(st[k]))
            h, w = sizes[k]
            _first_bad_row(n, frames[k, :h, :w], _oracle(family, n), _band(files[k]))
    # decode_jpeg: every size with its streams in one batch
    by_size = {}
    for n in names:
        by_size.setdefault(_hw(fn(n)), []).append(n)
    for hw, group in by_size.items():
        s, l = _pack([fn(n) for n in group])
        frames, status = data.decode_jpeg(s, l, hw)
        assert status.cpu().tolist() == [0] * len(group), group
        for k, n in enumerate(group):
            _first_bad_row(n, frames[k].cpu().numpy(), _oracle(family, n), _band(fn(n)))


@pytest.mark.gpu
def test_gpu_fixture_streams_equal_cv2():
    files = [FIX[n + ".jpg"].tobytes() for n in FIX_NAMES]
    sizes = [mks.CASES[n][:2] for n in FIX_NAMES]
    frames, st = _decode_sized_checked(files, sizes, (1200, 1920))
    for k, n in enumerate(FIX_NAMES):
        assert st[k] == 0, (n, jo.STATUS_NAMES.get(st[k]))
        h, w = sizes[k]
        _check_fixture(n, frames[k, :h, :w])
    for n, (h, w) in zip(FIX_NAMES, sizes):
        s, l = _pack([FIX[n + ".jpg"].tobytes()] * 2)
        frames, status = data.decode_jpeg(s, l, (h, w))
        assert status.cpu().tolist() == [0, 0], n
        for k in range(2):
            _check_fixture(n, frames[k].cpu().numpy())


@pytest.mark.gpu
def test_gpu_one_mixed_sized_launch():
    """every sampling, restart and self-synchronising streams, a 1 x 1 frame, a frame of the slot's size and a stream cut
    inside its scan in one decode_jpeg_sized launch"""
    slot = mks.CASES["s422_q90_opt_r7_45x77"][:2]
    items = [("fixture", "s422_q90_opt_r7_45x77"), ("generated", "g1x1_q1_smooth"), ("fixture", "s444_q80_40x72"),
             ("crafted", "units_2_16x32"), ("fixture", "s420_q85_r1000_33x65"), ("fixture", "s444_q95_r1_37x53"),
             ("generated", "g3x4_q88_flat"), ("rewritten", "fill_before_markers@s420_q90_31x47"),
             ("crafted", "units_1_8x8"), ("fixture", "s422_q75_32x64"), ("generated", "g16x32_q75_smooth")]
    files, sizes, want = [], [], []
    for fam, n in items:
        b = FIX[n + ".jpg"].tobytes() if fam == "fixture" else FAMILIES[fam][1](n)
        files.append(b)
        sizes.append(_hw(b))
        want.append(FIX[n + ".bgr"] if fam == "fixture" else _oracle(fam, n))
    assert sizes[0] == slot and all(h <= slot[0] and w <= slot[1] for h, w in sizes)
    cut = files[5][: len(files[5]) - 300]      # inside the restart intervals of a 4:4:4 stream
    files.insert(3, cut)
    sizes.insert(3, sizes[5])
    want.insert(3, None)
    assert jo.decode(cut)[1] == jo.EDATA
    frames, st = _decode_sized_checked(files, sizes, slot)
    for k, (h, w) in enumerate(sizes):
        if want[k] is None:
            assert st[k] == jo.EDATA, st
        else:
            assert st[k] == 0, (k, st[k])
            _first_bad_row(f"item {k}", frames[k, :h, :w], want[k], _band(files[k]))
