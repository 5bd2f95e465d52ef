"""The device path's Huffman decoding of sequential scans against files whose coefficients are known.

Every file here comes from tests/jpeg_writer.py, a baseline writer written from T.81, so the coefficients it
was given are the answer: read_jpeg must return them, and the device path (gb200_debug_entropy_decode_flags)
must return them too wherever it takes a file, at every subsequence size S.  The files reach what libjpeg never
writes: code lengths of 10 to 16 bits, table ids 2 and 3 and any table assignment, AC category 11, running DC
at the int16 edge on the 64-block chunk boundaries of the DC sums, restart intervals of every shape, and a
file that does not synchronise within the rounds allowed at S = 1024.  Each case is pinned to the path it takes
and the flags that send it there, so no case passes by going to the host.

On the GPU, the same hooks on the device, gb.decode_jpeg and gb.process_jpeg on tensors against the host-bytes
entries, Pillow's pixels, the route from the copy counters, and all the files in one call."""
import ctypes as C
import io
import zlib
from functools import lru_cache

import numpy as np
import pytest

import guetzli_b200 as gb
import jpeg_writer as jw

SEGMENT, CODE, RANGE, SYNC = gb.api.JPEG_BAD_SEGMENT, gb.api.JPEG_BAD_CODE, gb.api.JPEG_BAD_RANGE, gb.api.JPEG_BAD_SYNC
S_DEFAULT = 1024  # kJpegSubBits, pipeline.h
SIZES = [S_DEFAULT, 64, 33, 8]
SANE, INSANE, HOST = 1, 2, 0  # gb.api.jpeg_seed's routes


def max_rounds(S):
    return max(64, 65536 // S)  # jpeg_max_sync_rounds, pipeline.cu


# ---- the files ---------------------------------------------------------------------------------------------

def code_lengths(rng, symbols, lo, hi):
    """random code lengths in lo..hi (raised towards hi until they fit), the all-ones code left free"""
    while True:
        n = {s: int(rng.integers(lo, hi + 1)) for s in symbols}
        if sum(2.0 ** -k for k in n.values()) + 2.0 ** -max(n.values()) <= 1:
            return n
        lo = min(lo + 1, hi)


def random_tables(rng, lo, hi, ids=(0,)):
    t = {}
    for i in ids:
        t[(0, i)] = code_lengths(rng, jw.DC_SYMBOLS, lo, hi)
        t[(1, i)] = code_lengths(rng, jw.AC_SYMBOLS, lo, hi)
    return t


def random_coeffs(rng, w, h, comps, density=0.3, cats=(1, 6), dc=1023):
    """per component [blocks y][blocks x][64]: DC in -dc..dc, AC non-zero with the given density and categories"""
    out = []
    for bx, by in jw.mcu_grid(w, h, comps)[2]:
        a = np.zeros((by, bx, 64), np.int64)
        a[:, :, 0] = rng.integers(-dc, dc + 1, (by, bx))
        cat = rng.integers(cats[0], cats[1] + 1, (by, bx, 63))
        mag = (1 << (cat - 1)) + rng.integers(0, 1 << 11, (by, bx, 63)) % (1 << (cat - 1))
        a[:, :, 1:] = np.where(rng.random((by, bx, 63)) < density, rng.choice([-1, 1], (by, bx, 63)) * mag, 0)
        out.append(a)
    return out


def scan_blocks(w, h, comps, c, restart=0):
    """the (x, y) of component c's blocks in the order the scan codes them, one list per restart interval"""
    if len(comps) == 1:
        bx, by = jw.covered_blocks(w, h, comps, c)
        units = [[(x, y)] for y in range(by) for x in range(bx)]
    else:
        cols, rows, _ = jw.mcu_grid(w, h, comps)
        hc, vc = comps[c][:2]
        units = [[(mx * hc + ix, my * vc + iy) for iy in range(vc) for ix in range(hc)]
                 for my in range(rows) for mx in range(cols)]
    r = restart or len(units)
    return [sum(units[i:i + r], []) for i in range(0, len(units), r)]


def dc_spike(n, k, edge):
    """n running DC values that climb by 2047 (category 11) to `edge` at index k alone, then fall back"""
    d = np.abs(np.arange(n) - k)
    return np.sign(edge) * np.maximum(abs(edge) - 2047 * d, 0)


class Case:
    """One crafted file and what it must give: `taken` by the device path's shape, its status flags (one value,
    or {S: flags}), read_jpeg's error (None where it reads the file) and, where it does, the coefficients."""

    def __init__(self, name, make, flags=0, taken=True, read=None, seed=None, frame_order=True):
        self.name, self.make, self.taken, self.read = name, make, taken, read
        # T.81 B.2.3 lists a scan's components in frame order; libjpeg refuses a scan that does not
        self.frame_order = frame_order
        self.flags = flags if isinstance(flags, dict) else {S: flags for S in SIZES}
        self.seed = zlib.crc32(name.encode()) if seed is None else seed

    @lru_cache(maxsize=None)
    def file(self):
        """-> (bytes, coefficients read_jpeg lays out, frame components, quant tables)"""
        return self.make(np.random.default_rng(self.seed))

    def sizes(self):
        return SIZES if len(self.file()[0]) < 40000 else SIZES[:3]


CASES = {}


def case(name, **kw):
    def register(make):
        CASES[name] = Case(name, make, **kw)
        return make
    return register


def crafted(w, h, comps, tables, coeffs, **writer):
    b = jw.write_jpeg(w, h, comps, coeffs, tables, **writer)
    return b, jw.scan_coefficients(w, h, comps, coeffs), comps, writer.get("quant")


def simple(name, w, h, comps, lo, hi, ids=(0,), coeff_kw=None, flags=0, taken=True, read=None, seed=None,
           **writer):
    """a case of random tables with lengths lo..hi under `ids` and random coefficients"""
    def make(rng):
        tables = random_tables(rng, lo, hi, ids)
        return crafted(w, h, comps, tables, random_coeffs(rng, w, h, comps, **(coeff_kw or {})), **writer)
    order = writer.get("scan_order")
    CASES[name] = Case(name, make, flags=flags, taken=taken, read=read, seed=seed,
                       frame_order=order is None or list(order) == sorted(order))


P444, P422, P420 = [(1, 1)] * 3, [(2, 1), (1, 1), (1, 1)], [(2, 2), (1, 1), (1, 1)]


def comps_of(sampling, tabs):
    return [s + t for s, t in zip(sampling, tabs)]


# -- code lengths
simple("len16 444", 40, 24, comps_of(P444, [(0, 0)] * 3), 16, 16)
simple("len16 420 rst3", 35, 20, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 16, 16, ids=(0, 1), restart=3)
simple("len9-16 444", 61, 45, comps_of(P444, [(0, 0)] * 3), 9, 16, coeff_kw={"density": 0.4})
simple("len9-16 420 rst5", 77, 53, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 9, 16, ids=(0, 1), restart=5)
simple("len9-16 gray", 45, 37, [(1, 1, 0, 0)], 9, 16)


@case("len1-3 stuffing 444", flags=RANGE)
def _(rng):
    """codes of 1 to 3 bits and category-10 values of all 1-bits: 0xFF data bytes, stuffed, almost everywhere"""
    w, h = 48, 32
    comps = comps_of(P444, [(0, 0)] * 3)
    tables = {(0, 0): {0: 1, 1: 2}, (1, 0): {0x0A: 1, jw.EOB: 2, 0x1A: 3}}
    co = []
    for bx, by in jw.mcu_grid(w, h, comps)[2]:
        a = np.zeros((by, bx, 64), np.int64)
        a[:, :, 0] = 1
        for y in range(by):
            for x in range(bx):
                k = 1
                while k < 56 and rng.random() < 0.9:
                    k += int(rng.random() < 0.25)
                    a[y, x, jw.ZIGZAG[k]] = 1023
                    k += 1
        co.append(a)
    out = crafted(w, h, comps, tables, co)
    assert out[0].count(b"\xff\x00") > len(out[0]) // 8, "the file is not dense in stuffed bytes"
    return out


@case("dc one symbol 444")
def _(rng):
    """a DC table with one symbol (category 0): every DC value 0"""
    w, h = 33, 25
    comps = comps_of(P444, [(0, 0)] * 3)
    tables = {(0, 0): {0: 1}, (1, 0): code_lengths(rng, jw.AC_SYMBOLS, 4, 12)}
    co = random_coeffs(rng, w, h, comps)
    for a in co:
        a[:, :, 0] = 0
    return crafted(w, h, comps, tables, co)


def every_ac_symbol_blocks(rng, nblocks):
    """blocks whose coding uses every AC symbol: run 0..15 with size 1..11, ZRL and EOB"""
    pairs = [(r, s) for r in range(16) for s in range(1, 12)]
    rng.shuffle(pairs)
    blocks, blk, k = [], np.zeros(64, np.int64), 1
    for r, s in pairs:
        if k + r > 63:
            blocks.append(blk)
            blk, k = np.zeros(64, np.int64), 1
        blk[jw.ZIGZAG[k + r]] = int(rng.choice([-1, 1])) * int(rng.integers(1 << (s - 1), 1 << s))
        k += r + 1
    blocks.append(blk)
    zrl = np.zeros(64, np.int64)
    zrl[jw.ZIGZAG[40]] = 3  # ZRL, ZRL, then run 7
    blocks.append(zrl)
    while len(blocks) < nblocks:
        blocks.append(np.zeros(64, np.int64))
    for b in blocks:
        b[0] = int(rng.integers(-500, 500))
    return np.array(blocks[:nblocks])


def ac_symbols_used(blocks):
    used = set()
    for blk in blocks:
        zz = [int(blk[jw.ZIGZAG[k]]) for k in range(64)]
        last = max([k for k in range(1, 64) if zz[k]], default=0)
        run = 0
        for k in range(1, last + 1):
            if not zz[k]:
                run += 1
                continue
            while run > 15:
                used.add(jw.ZRL)
                run -= 16
            used.add((run << 4) | jw.category(zz[k]))
            run = 0
        if last < 63:
            used.add(jw.EOB)
    return used


@case("ac 178 symbols gray", flags=RANGE)
def _(rng):
    w, h = 64, 40
    comps = [(1, 1, 0, 0)]
    tables = {(0, 0): code_lengths(rng, jw.DC_SYMBOLS, 2, 9), (1, 0): code_lengths(rng, jw.AC_SYMBOLS, 8, 16)}
    blocks = every_ac_symbol_blocks(rng, 40)
    assert ac_symbols_used(blocks) == set(jw.AC_SYMBOLS)
    return crafted(w, h, comps, tables, [blocks.reshape(5, 8, 64)])


# -- table layouts: period 1 and period nslot (3, 4, 6), AC-only differences, ids 2 and 3, luma on the chroma
# pair, tables with different ids and the same codes, scan orders other than the frame's
LAYOUTS = {
    "444": (P444, 41, 27, [
        ("p1", [(0, 0)] * 3), ("p3", [(0, 0), (1, 1), (1, 1)]), ("p3 ac only", [(0, 0), (0, 1), (0, 1)]),
        ("p3 dc only", [(0, 0), (1, 0), (1, 0)]), ("ids 2 3", [(2, 3), (3, 2), (2, 2)]),
        ("luma on chroma", [(1, 1), (0, 0), (0, 0)])]),
    "422": (P422, 50, 30, [
        ("p1", [(1, 1)] * 3), ("p4", [(0, 0), (1, 1), (1, 1)]), ("p4 y cr share", [(0, 0), (1, 1), (0, 0)]),
        ("p4 ac only", [(0, 0), (0, 1), (0, 1)]), ("ids 3 2", [(3, 3), (2, 2), (2, 2)])]),
    "420": (P420, 77, 53, [
        ("p1", [(0, 0)] * 3), ("p6", [(0, 0), (1, 1), (1, 1)]), ("p6 ac only", [(0, 0), (0, 1), (0, 1)]),
        ("p6 cb differs", [(0, 0), (1, 1), (0, 0)]), ("ids 0-3", [(2, 3), (1, 0), (3, 2)]),
        ("luma on chroma", [(1, 1), (0, 0), (0, 0)])]),
}
for sub, (sampling, W, H, assignments) in LAYOUTS.items():
    for label, tabs in assignments:
        simple(f"layout {sub} {label}", W, H, comps_of(sampling, tabs), 4, 14, ids=(0, 1, 2, 3))
simple("layout 444 scan order 2 0 1", 41, 27, comps_of(P444, [(0, 0), (1, 1), (0, 1)]), 4, 14, ids=(0, 1),
       scan_order=[2, 0, 1])
simple("layout 420 scan order 1 2 0 rst4", 77, 53, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 4, 14, ids=(0, 1),
       scan_order=[1, 2, 0], restart=4)
simple("layout gray id 3", 30, 20, [(1, 1, 3, 3)], 4, 14, ids=(3,))
simple("layout 444 one dht per table", 41, 27, comps_of(P444, [(0, 0), (1, 1), (1, 1)]), 4, 14, ids=(0, 1),
       dht_per_table=True)


@case("layout 420 same codes under ids 0 and 2")
def _(rng):
    """Y on tables 0, Cb on tables 2 with the same codes, Cr on tables 1: the decoder merges 0 and 2"""
    w, h = 77, 53
    tables = random_tables(rng, 4, 14, (0, 1))
    tables[(0, 2)], tables[(1, 2)] = dict(tables[(0, 0)]), dict(tables[(1, 0)])
    comps = comps_of(P420, [(0, 0), (2, 2), (1, 1)])
    return crafted(w, h, comps, tables, random_coeffs(rng, w, h, comps))


@case("layout 444 same codes under ids 1 and 3")
def _(rng):
    """every component on tables with the same codes under two ids: period 1 once merged"""
    w, h = 41, 27
    tables = random_tables(rng, 4, 14, (1,))
    tables[(0, 3)], tables[(1, 3)] = dict(tables[(0, 1)]), dict(tables[(1, 1)])
    comps = comps_of(P444, [(1, 3), (3, 1), (1, 1)])
    return crafted(w, h, comps, tables, random_coeffs(rng, w, h, comps))


# -- coefficients
simple("ac cat 10 11 444", 33, 17, comps_of(P444, [(0, 0), (1, 1), (1, 1)]), 5, 14, ids=(0, 1),
       coeff_kw={"density": 0.05, "cats": (10, 11)}, flags=RANGE)
simple("ac cat 11 gray dense", 24, 16, [(1, 1, 0, 0)], 9, 16, coeff_kw={"density": 0.5, "cats": (11, 11)},
       flags=RANGE)


@case("ac cat 11 sparse 444")
def _(rng):
    """one category-11 coefficient per block of small ones, at |coef| = 1024 and 2047"""
    w, h = 40, 24
    comps = comps_of(P444, [(0, 0)] * 3)
    co = random_coeffs(rng, w, h, comps, density=0.1, cats=(1, 2), dc=100)
    for c, a in enumerate(co):
        a[:, :, jw.ZIGZAG[1 + 20 * c]] = np.where(np.arange(a.shape[1]) % 2, 1024, -2047)
    return crafted(w, h, comps, random_tables(rng, 3, 16), co)


@case("dc cat 11 444")
def _(rng):
    """running DC alternating between 1023 and -1024: every difference of category 11"""
    w, h = 40, 24
    comps = comps_of(P444, [(0, 0), (1, 1), (1, 1)])
    co = random_coeffs(rng, w, h, comps, density=0.1, cats=(1, 3))
    for a in co:
        a[:, :, 0] = np.where((np.arange(a.shape[0])[:, None] + np.arange(a.shape[1])) % 2, 1023, -1024)
    return crafted(w, h, comps, random_tables(rng, 3, 16, (0, 1)), co)


@case("zrl chains 444")
def _(rng):
    """blocks whose only AC coefficient is at zig-zag 16, 17, 32, 33, 48, 49 or 63: chains of 1 to 3 ZRLs"""
    w, h = 56, 16
    comps = comps_of(P444, [(0, 0)] * 3)
    co = random_coeffs(rng, w, h, comps, density=0.0)
    spots = [16, 17, 32, 33, 48, 49, 63]
    for a in co:
        for y in range(a.shape[0]):
            for x in range(a.shape[1]):
                a[y, x, jw.ZIGZAG[spots[(x + y) % len(spots)]]] = int(rng.integers(1, 300)) * int(rng.choice([-1, 1]))
    return crafted(w, h, comps, random_tables(rng, 2, 12), co)


@case("full blocks 444")
def _(rng):
    """every coefficient of every block non-zero: no block has an EOB"""
    w, h = 24, 24
    comps = comps_of(P444, [(0, 0), (1, 1), (1, 1)])
    co = random_coeffs(rng, w, h, comps, density=1.0, cats=(1, 3))
    return crafted(w, h, comps, random_tables(rng, 3, 14, (0, 1)), co)


# -- DC sums at the int16 edge, on the chunk boundaries (kJpegDcChunk = 64) of one (interval, component) task
DC_ACCEPTED, DC_REFUSED = (32767, -32768), (32768, -32769)


def dc_edge_case(name, sampling, w, h, c, k, edge, restart=0, interval=0):
    def make(rng):
        comps = comps_of(sampling, [(0, 0)] * len(sampling))
        co = random_coeffs(rng, w, h, comps, density=0.02, cats=(1, 2), dc=0)
        blocks = scan_blocks(w, h, comps, c, restart)[interval]
        for (x, y), v in zip(blocks, dc_spike(len(blocks), k, edge)):
            co[c][y, x, 0] = v
        return crafted(w, h, comps, {(0, 0): code_lengths(rng, jw.DC_SYMBOLS, 2, 8),
                                     (1, 0): code_lengths(rng, jw.AC_SYMBOLS, 3, 12)}, co, restart=restart)
    # a DC value near the int16 edge is far outside the SIMD IDCT's range, so the range test flags every file
    refused = edge in DC_REFUSED
    CASES[name] = Case(name, make, flags=CODE | RANGE if refused else RANGE,
                       read="Invalid DC coefficient" if refused else None)


for k in (63, 64, 65, 128):
    for edge in DC_ACCEPTED + DC_REFUSED:
        dc_edge_case(f"dc edge gray k={k} {edge:+d}", [(1, 1)], 8 * 140, 8, 0, k, edge)
        # 4:2:0, Y and Cb blocks interleaved: the k-th block of Y, then of Cb (one per MCU)
        dc_edge_case(f"dc edge 420 y k={k} {edge:+d}", P420, 16 * 40, 16, 0, k, edge)
        dc_edge_case(f"dc edge 420 cb k={k} {edge:+d}", P420, 16 * 130, 16, 1, k, edge)
    for edge in (32767, 32768, -32769):
        # in the second restart interval, which starts a task and a chunk count of its own
        dc_edge_case(f"dc edge gray rst k={k} {edge:+d}", [(1, 1)], 8 * 300, 8, 0, k, edge, restart=140, interval=1)
        dc_edge_case(f"dc edge 420 cr rst k={k} {edge:+d}", P420, 16 * 300, 16, 2, k, edge, restart=140, interval=1)

# -- shapes: sizes that are and are not multiples of the MCU, restart intervals, single components with
# sampling factors
for sub, sampling in [("444", P444), ("422", P422), ("420", P420)]:
    for w, h in [(1, 1), (8, 8), (9, 7), (16, 16), (17, 15), (33, 17)]:
        simple(f"size {sub} {w}x{h}", w, h, comps_of(sampling, [(0, 0), (1, 1), (1, 1)]), 2, 12, ids=(0, 1))
for f, w, h in [((1, 1), 1, 1), ((1, 1), 13, 9), ((2, 2), 1, 1), ((2, 2), 37, 29), ((2, 1), 21, 13),
                ((1, 2), 19, 23), ((2, 2), 16, 16)]:
    simple(f"size gray {f[0]}x{f[1]} {w}x{h}", w, h, [f + (0, 0)], 2, 12)
for R in (1, 2, 3, 4, 8, 9, 10, 1000):  # 9 MCUs: 2 and 4 do not divide them
    simple(f"restart 420 40x40 R={R}", 40, 40, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 3, 16, ids=(0, 1),
           restart=R)
for R in (1, 3, 19, 20, 21):  # 20 non-interleaved MCUs
    simple(f"restart gray 2x2 37x29 R={R}", 37, 29, [(2, 2, 0, 0)], 3, 16, restart=R)
simple("restart 444 R=1 long codes", 33, 17, comps_of(P444, [(0, 0)] * 3), 12, 16, restart=1,
       coeff_kw={"density": 0.5})
simple("restart 444 R=7 sof1", 57, 41, comps_of(P444, [(0, 0), (1, 1), (1, 1)]), 3, 16, ids=(0, 1), restart=7,
       sof=0xC1)
# libjpeg_decodable's layouts only: 2x1 on every component is read by read_jpeg and refused by the device shape
simple("shape 444 all 2x1", 50, 30, comps_of([(2, 1)] * 3, [(0, 0)] * 3), 3, 12, taken=False)

# -- stream variants libjpeg does not write
simple("stream zrl to 63 444", 40, 24, comps_of(P444, [(0, 0)] * 3), 3, 14, trailing_zrl=True,
       coeff_kw={"density": 0.08})
simple("stream zero padding 420 rst2", 40, 40, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 3, 14, ids=(0, 1),
       restart=2, pad_bit=0)
simple("stream zero padding gray", 21, 13, [(1, 1, 0, 0)], 3, 14, pad_bit=0)
simple("stream bytes before eoi 444", 40, 24, comps_of(P444, [(0, 0)] * 3), 3, 14, tail=b"\x00\x12\x34\xfe")
simple("stream bytes before eoi 420 rst3", 40, 40, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 3, 14, ids=(0, 1),
       restart=3, tail=b"\x55" * 9)
# fill bytes: read_jpeg skips them before EOI and refuses them before RSTn; the segment pass sends both to the host
simple("stream fill before eoi 444", 40, 24, comps_of(P444, [(0, 0)] * 3), 3, 14, fill_bytes=2, flags=SEGMENT)
simple("stream fill before rst 420", 40, 40, comps_of(P420, [(0, 0), (1, 1), (1, 1)]), 3, 14, ids=(0, 1),
       restart=3, fill_bytes=1, flags=SEGMENT | CODE, read="Did not find expected restart marker")

# -- files that do not synchronise within jpeg_max_sync_rounds(1024) = 64 rounds: long codes, dense
# coefficients, one restart interval of ~95 and ~255 subsequences; they do at smaller S.  The write pass from
# the states of the last round then fails as well (kJpegBadCode).
for (w, h), seed in [((64, 48), 4), ((128, 64), 0)]:
    simple(f"sync 444 {w}x{h}", w, h, comps_of(P444, [(0, 0)] * 3), 12, 16, seed=seed,
           coeff_kw={"density": 0.6, "cats": (1, 4)}, flags={1024: SYNC | CODE, 64: 0, 33: 0, 8: 0})

NAMES = sorted(CASES)
ACCEPTED = [n for n in NAMES if CASES[n].read is None]


def frame_444(n):
    comps = CASES[n].file()[2]
    return len(comps) == 3 and all(c[:2] == (1, 1) for c in comps)


CASES_444 = [n for n in NAMES if frame_444(n)]


# ---- CPU port ----------------------------------------------------------------------------------------------

def check_case(lib, name, sizes):
    """read_jpeg gives the writer's coefficients (or its pinned error); the device path takes the file and flags
    it as pinned, with the writer's coefficients wherever it keeps the file"""
    c = CASES[name]
    b, truth, _, _ = c.file()
    ok, _, got = gb.api.read_jpeg(b, lib=lib)
    if c.read is None:
        assert ok and np.array_equal(got, truth), f"{name}: read_jpeg differs from the writer's coefficients"
    else:
        assert not ok and gb.last_error(lib=lib) == c.read, (name, gb.last_error(lib=lib))
    for S in sizes:
        taken, flags, rounds, coeffs = gb.api.entropy_decode_flags(b, S, lib=lib)
        assert (taken, flags) == (c.taken, c.flags[S] if c.taken else 0), (name, S, taken, flags)
        assert rounds <= max_rounds(S), (name, S, rounds)
        if flags & SYNC:
            assert rounds == max_rounds(S), (name, S, rounds)
        if taken and not flags & ~RANGE:
            assert np.array_equal(coeffs[:truth.size], truth), f"{name} S={S}: coefficients differ"
            assert not coeffs[truth.size:truth.size + 4096].any(), f"{name} S={S}: written beyond the coefficients"
        # the existing hook tells the same story
        t, c2 = gb.api.entropy_decode(b, S, lib=lib)
        assert t == (taken and not flags & ~RANGE), (name, S)
        if t:
            assert np.array_equal(c2[:truth.size], truth), (name, S)


@pytest.mark.parametrize("name", NAMES)
def test_port_crafted(port_lib, name):
    check_case(port_lib, name, CASES[name].sizes())


def seed_expectation(c, S):
    """the route and plane gb200_debug_jpeg_seed must give for a 4:4:4 case"""
    b, truth, comps, quant = c.file()
    quant = quant or {0: [1] * 64}
    q = np.array([quant[comp[4] if len(comp) > 4 else 0] for comp in comps], np.int64)
    if c.read is not None or (c.flags[S] & ~RANGE):
        return HOST, None
    v = truth.reshape(3, -1, 64) * q[:, None, :]
    return (SANE if np.abs(v).max() <= 4096 else INSANE), v.reshape(-1)


def check_seed(lib, c, S):
    """the seeding of process_jpeg's device route gives the writer's coefficients times their quant steps, and
    the sanity verdict on them, wherever the pinned flags let the route take the file -> route"""
    want, v = seed_expectation(c, S)
    route, dq = gb.api.jpeg_seed(c.file()[0], S, lib=lib)
    assert route == want, (c.name, S, route, want)
    if route != HOST:
        assert np.array_equal(dq[:v.size], v.astype(np.int16)), f"{c.name} S={S}: dq differs"
        assert not dq[v.size:v.size + 4096].any(), f"{c.name} S={S}: written beyond the plane"
    return route


@pytest.mark.parametrize("S", [S_DEFAULT, 33])
def test_port_seed_444(port_lib, S):
    routes = [check_seed(port_lib, CASES[name], S) for name in CASES_444]
    assert routes.count(SANE) > len(routes) // 2 and HOST in routes


def ac11_at_bound(coef, step, k=9):
    """a 4:4:4 file with AC coefficient `coef` (category 11) at natural index k of every Y block, quant step
    `step` there"""
    def make(rng):
        w, h = 24, 16
        comps = [(1, 1, 0, 0, 1), (1, 1, 0, 0, 0), (1, 1, 0, 0, 0)]
        co = random_coeffs(rng, w, h, comps, density=0.1, cats=(1, 3), dc=200)
        co[0][:, :, k] = coef
        q = [1] * 64
        q[k] = step
        return crafted(w, h, comps, random_tables(rng, 3, 16), co, quant={0: [1] * 64, 1: q})
    return Case(f"ac11 {coef}x{step}", make)


@pytest.mark.parametrize("coef, step, want", [(1024, 4, SANE), (-1024, 4, SANE), (1025, 4, INSANE),
                                              (-1025, 4, INSANE), (2047, 2, SANE), (2047, 3, INSANE)])
def test_port_seed_ac11_bound(port_lib, coef, step, want):
    """|coef * q| = 4096 passes the sanity bound and 4100 does not, with AC coefficients of category 11"""
    c = ac11_at_bound(coef, step)
    for S in (S_DEFAULT, 8):
        assert check_seed(port_lib, c, S) == want


# ---- on the GPU --------------------------------------------------------------------------------------------

def on_device(b, dev="cuda:0"):
    import torch
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)


def host_decode(lib, b):
    """the host-bytes entry -> pixels, or its reason for refusing"""
    try:
        return gb.decode_jpeg(b, cuda=False, lib=lib)
    except ValueError as e:
        return str(e).split(": file 0: ", 1)[1]


@pytest.mark.gpu
def test_cuda_hooks(cuda_lib):
    """the hooks on the device give the port's routes, flags and coefficients"""
    for name in NAMES:
        check_case(cuda_lib, name, [S_DEFAULT, 33])


@pytest.mark.gpu
def test_cuda_seed_444(cuda_lib):
    for name in CASES_444:
        for S in (S_DEFAULT, 33):
            check_seed(cuda_lib, CASES[name], S)


MAX_STATUS_BYTES = 4 * (64 + 2)


@pytest.mark.gpu
def test_cuda_decode_from_tensors(cuda_lib):
    """gb.decode_jpeg on a tensor gives the host-bytes entry's pixels or refusal, by the pinned route: the device
    path copies back the header prefix and status words, the host path the whole file"""
    for name in NAMES:
        c = CASES[name]
        b = c.file()[0]
        want = host_decode(cuda_lib, b)
        _, _, d0 = gb.counters(lib=cuda_lib)
        try:
            got = gb.decode_jpeg(on_device(b), lib=cuda_lib).cpu().numpy()
        except ValueError as e:
            got = str(e).split(": file 0: ", 1)[1]
        _, _, d1 = gb.counters(lib=cuda_lib)
        if isinstance(want, str):
            assert got == want, (name, got, want)
        else:
            assert isinstance(got, np.ndarray) and np.array_equal(got, want), name
        extra = d1 - d0 - 2 * min(4096, len(b))
        if c.taken and c.flags[S_DEFAULT] == 0:
            assert extra <= MAX_STATUS_BYTES, (name, extra)
        else:
            assert extra >= len(b), (name, extra)


@pytest.mark.gpu
def test_cuda_against_pillow(cuda_lib):
    """Pillow (libjpeg-turbo) reads every file the host entry accepts to the same pixels, and the SIMD-range test
    refuses the files the device flagged for it.  (Scans whose components are not in frame order are read by
    read_jpeg, as by ReadJpeg, and refused by libjpeg: DESIGN.md section 8.)"""
    Image = pytest.importorskip("PIL.Image", reason="Pillow decodes the files")
    accepted = 0
    for name in [n for n in ACCEPTED if CASES[n].frame_order]:
        b = CASES[name].file()[0]
        want = host_decode(cuda_lib, b)
        if isinstance(want, str):
            # refused for a sampling the decoder does not take (DESIGN.md section 8), or by the SIMD-range test
            if not CASES[name].taken:
                assert want.startswith("sampling factors ") and "are decoded" in want, (name, want)
            else:
                assert CASES[name].flags[S_DEFAULT] & RANGE and "SIMD IDCT" in want, (name, want)
            continue
        assert not CASES[name].flags[S_DEFAULT] & RANGE or not CASES[name].taken, name
        px = np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))
        assert np.array_equal(px, want), name
        accepted += 1
    assert accepted > len(ACCEPTED) // 2


def raw_from_device(lib, files, shapes, sentinel):
    import torch
    n = len(files)
    out = [torch.full(s, sentinel, dtype=torch.uint8, device="cuda:0") for s in shapes]
    ok = lib.gb200_jpeg_decode_rgb_from_device(
        (C.c_void_p * n)(*[f.data_ptr() for f in files]), (C.c_size_t * n)(*[f.numel() for f in files]), n, 0,
        (C.c_int * n)(*[s[1] for s in shapes]), (C.c_int * n)(*[s[0] for s in shapes]),
        (C.c_void_p * n)(*[o.data_ptr() for o in out]), torch.cuda.current_stream().cuda_stream)
    return ok, out


@pytest.mark.gpu
def test_cuda_one_call(cuda_lib):
    """every file the host entry accepts in one call from tensors, device-path, unsynchronised and host-shape
    files mixed: each comes out as alone; then one refused file in the middle is refused by its index and no
    output is written"""
    files, wants = [], []
    for name in ACCEPTED:
        want = host_decode(cuda_lib, CASES[name].file()[0])
        if not isinstance(want, str):
            files.append(CASES[name].file()[0])
            wants.append(want)
    assert any(CASES[n].flags[S_DEFAULT] & SYNC for n in ACCEPTED)
    out = gb.decode_jpeg([on_device(b) for b in files], lib=cuda_lib)
    for b, px, want in zip(files, out, wants):
        assert np.array_equal(px.cpu().numpy(), want)
    bad = CASES["dc edge 420 cb k=64 +32768"].file()[0]
    mid = len(files) // 2
    mixed = files[:mid] + [bad] + files[mid:]
    with pytest.raises(ValueError) as e:
        gb.decode_jpeg([on_device(b) for b in mixed], lib=cuda_lib)
    assert str(e.value) == f"jpeg_decode_rgb_from_device: file {mid}: Invalid DC coefficient"
    shapes = [w.shape for w in wants[:mid]] + [(16, 16 * 130, 3)] + [w.shape for w in wants[mid:]]
    ok, outs = raw_from_device(cuda_lib, [on_device(b) for b in mixed], shapes, 201)
    assert not ok and gb.last_error(lib=cuda_lib) == str(e.value)
    assert all(bool((o == 201).all()) for o in outs)


@pytest.mark.gpu
def test_cuda_process_jpeg_444(cuda_lib):
    """gb.process_jpeg on tensors gives the host-bytes entry's outcome for the 4:4:4 files, by the pinned route"""
    from test_process_jpeg_from_device import MAX_STATUS_BYTES as SEED_STATUS_BYTES, same_as_host
    for name in CASES_444:
        b = CASES[name].file()[0]
        dev, host = same_as_host(cuda_lib, b, 90, name=name)
        extra = dev["d2h_bytes"] - host["d2h_bytes"]
        if seed_expectation(CASES[name], S_DEFAULT)[0] != HOST:
            assert 0 < extra <= 2 * 4096 + SEED_STATUS_BYTES, (name, extra)
        else:
            assert extra >= len(b), (name, extra)
