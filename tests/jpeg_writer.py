"""A baseline JPEG writer for tests: quantised coefficients in, a sequential Huffman-coded file out.

Written from ITU-T T.81: the marker segments of Annex B, the Huffman code generation of Annex C and the
sequential encoding procedures of F.1.2.  It knows nothing of the decoder under test, so the coefficients it
is given are the known answer for the file it writes.  Unlike an encoder it takes any Huffman code lengths,
any table assignment and component order, any sampling factors and restart interval, and a few stream
variants that the format allows but libjpeg does not write (see `write_jpeg`).
"""
import numpy as np

# natural (row-major) index of each zig-zag position (T.81 Figure A.6)
ZIGZAG = sorted(range(64), key=lambda i: (i // 8 + i % 8, (i % 8) if (i // 8 + i % 8) % 2 == 0 else i // 8))

EOB, ZRL = 0x00, 0xF0
DC_SYMBOLS = list(range(12))
# every AC symbol a sequential 8-bit scan can use: EOB, ZRL, and run 0..15 with size 1..11
AC_SYMBOLS = [EOB, ZRL] + [(r << 4) | s for r in range(16) for s in range(1, 12)]


def canonical_codes(lengths):
    """{symbol: code length in 1..16} -> (BITS[16], HUFFVAL, {symbol: (code, length)}).

    HUFFVAL lists the symbols by code length, then by value; the codes follow Annex C (Figures C.1 to C.3):
    consecutive integers within a length, shifted left by one for each longer length.  No code may be all
    1-bits (C.2), so the lengths must leave room for that."""
    if not lengths:
        raise ValueError("a Huffman table needs at least one symbol")
    for s, n in lengths.items():
        if not 1 <= n <= 16:
            raise ValueError(f"symbol {s:#x}: code length {n} is not in 1..16")
    huffval = sorted(lengths, key=lambda s: (lengths[s], s))
    bits = [sum(1 for n in lengths.values() if n == k) for k in range(1, 17)]
    codes, code, k = {}, 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            codes[huffval[k]] = (code, n)
            code += 1
            k += 1
        code <<= 1
    for s, (c, n) in codes.items():
        if c >= (1 << n) - 1:
            raise ValueError(f"symbol {s:#x}: the lengths leave no room for a code of {n} bits that is not all "
                             "1-bits")
    return bits, huffval, codes


def category(v):
    """SSSS of a value (T.81 Table F.1 / F.2): its magnitude's bit length"""
    return int(abs(int(v))).bit_length()


def magnitude_bits(v, s):
    """the s additional bits of a value (F.1.2.1.1): v itself when positive, v - 1 in s bits when negative"""
    return v if v >= 0 else v + (1 << s) - 1


class BitWriter:
    """MSB-first entropy-coded segment with 0xFF stuffing (F.1.2.3)"""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, value, n):
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((value >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0x00)
                self.acc = self.n = 0

    def pad(self, bit):
        """fill the last byte with `bit` (F.1.2.3 asks for 1-bits)"""
        while self.n:
            self.put(bit, 1)

    def take(self):
        b = bytes(self.out)
        self.out = bytearray()
        return b


def segment(marker, payload):
    n = len(payload) + 2
    return bytes([0xFF, marker, n >> 8, n & 255]) + bytes(payload)


def encode_block(bw, blk, prev_dc, dc_codes, ac_codes, trailing_zrl=False):
    """one block (64 coefficients in natural order) after F.1.2.1 and F.1.2.2 -> its DC value.

    trailing_zrl: where the zeros after the last non-zero coefficient fill whole runs of 16 up to index 63,
    code them as ZRLs (the block then ends at index 63 without an EOB) instead of as an EOB."""
    zz = [int(blk[ZIGZAG[k]]) for k in range(64)]
    diff = zz[0] - prev_dc
    s = category(diff)
    if s > 11:
        raise ValueError(f"DC difference {diff} is beyond category 11")
    code(bw, dc_codes, s)
    bw.put(magnitude_bits(diff, s), s)
    run = 0
    last = max([k for k in range(1, 64) if zz[k]], default=0)
    for k in range(1, last + 1):
        if zz[k] == 0:
            run += 1
            continue
        while run > 15:
            code(bw, ac_codes, ZRL)
            run -= 16
        s = category(zz[k])
        if s > 11:
            raise ValueError(f"AC value {zz[k]} is beyond category 11")
        code(bw, ac_codes, (run << 4) | s)
        bw.put(magnitude_bits(zz[k], s), s)
        run = 0
    if last < 63:
        if trailing_zrl and (63 - last) % 16 == 0:
            for _ in range((63 - last) // 16):
                code(bw, ac_codes, ZRL)
        else:
            code(bw, ac_codes, EOB)
    return zz[0]


def code(bw, codes, symbol):
    if symbol not in codes:
        raise ValueError(f"symbol {symbol:#04x} has no code in its table")
    bw.put(*codes[symbol])


def mcu_grid(width, height, comps):
    """(MCU columns, MCU rows) of an interleaved scan (A.2.3), and each component's blocks (x, y) padded to it"""
    hmax = max(c[0] for c in comps)
    vmax = max(c[1] for c in comps)
    cols, rows = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    return cols, rows, [(cols * c[0], rows * c[1]) for c in comps]


def covered_blocks(width, height, comps, c):
    """blocks (x, y) of component c that a scan of it alone covers (A.2.2): the component's own size in blocks"""
    hmax = max(k[0] for k in comps)
    vmax = max(k[1] for k in comps)
    cw = -(-width * comps[c][0] // hmax)
    ch = -(-height * comps[c][1] // vmax)
    return -(-cw // 8), -(-ch // 8)


def write_jpeg(width, height, comps, coeffs, tables, restart=0, sof=0xC0, scan_order=None, quant=None,
               pad_bit=1, fill_bytes=0, tail=b"", trailing_zrl=False, dht_per_table=False):
    """A baseline (sof=0xC0) or extended sequential (0xC1) file with one scan carrying every component.

    comps: per frame component (H, V, DC table id, AC table id) or (H, V, DC id, AC id, Tq); component ids are
        1, 2, ... in frame order.
    coeffs: per frame component, an integer array [blocks y][blocks x][64] of quantised coefficients in natural
        order, padded to the MCU grid (mcu_grid).  A one-component scan is not interleaved (A.2.2): it codes
        the component's own blocks (covered_blocks) and the padding blocks are not in the file.
    tables: {(0 for DC | 1 for AC, table id 0..3): {symbol: code length}}; written in that order.
    restart: the restart interval in MCUs (DRI), 0 for none; RSTn cycle through 0..7.
    scan_order: frame component indices in the order the scan header lists them (default frame order; T.81
        B.2.3 asks for frame order, and libjpeg refuses any other).
    quant: {Tq: 64 quantisation steps in natural order}; default one table 0 of all 1s.

    Stream variants: pad_bit, the bit that fills the byte before each RSTn and before EOI (F.1.2.3 asks for 1);
    fill_bytes, that many 0xFF fill bytes (B.1.1.2) before each RSTn and before EOI; tail, bytes between the
    last MCU's data and EOI; trailing_zrl, see encode_block; dht_per_table, one DHT segment per table instead
    of one for all."""
    n = len(comps)
    comps = [tuple(c) + (0,) * (5 - len(c)) for c in comps]
    order = list(range(n)) if scan_order is None else list(scan_order)
    quant = {0: [1] * 64} if quant is None else quant
    out = bytearray(b"\xFF\xD8")
    for tq in sorted(quant):
        q = [int(quant[tq][ZIGZAG[k]]) for k in range(64)]
        if max(q) > 255:
            out += segment(0xDB, [0x10 | tq] + sum([[v >> 8, v & 255] for v in q], []))
        else:
            out += segment(0xDB, [tq] + q)
    out += segment(sof, [8, height >> 8, height & 255, width >> 8, width & 255, n] +
                   sum([[c + 1, (comps[c][0] << 4) | comps[c][1], comps[c][4]] for c in range(n)], []))
    codes, dht = {}, []
    for (cls, tid), lengths in tables.items():
        bits, huffval, codes[(cls, tid)] = canonical_codes(lengths)
        dht.append([(cls << 4) | tid] + bits + huffval)
    if dht_per_table:
        for t in dht:
            out += segment(0xC4, t)
    else:
        out += segment(0xC4, sum(dht, []))
    if restart:
        out += segment(0xDD, [restart >> 8, restart & 255])
    out += segment(0xDA, [len(order)] + sum([[c + 1, (comps[c][2] << 4) | comps[c][3]] for c in order], []) +
                   [0, 63, 0])

    if len(order) == 1:
        c = order[0]
        bx, by = covered_blocks(width, height, comps, c)
        units = [[(c, x, y)] for y in range(by) for x in range(bx)]
    else:
        cols, rows, _ = mcu_grid(width, height, comps)
        units = [[(c, mx * comps[c][0] + ix, my * comps[c][1] + iy)
                  for c in order for iy in range(comps[c][1]) for ix in range(comps[c][0])]
                 for my in range(rows) for mx in range(cols)]
    bw = BitWriter()
    pred = [0] * n
    for m, unit in enumerate(units):
        if restart and m and m % restart == 0:
            bw.pad(pad_bit)
            out += bw.take() + b"\xFF" * fill_bytes + bytes([0xFF, 0xD0 + (m // restart - 1) % 8])
            pred = [0] * n
        for c, x, y in unit:
            dc_codes, ac_codes = codes[(0, comps[c][2])], codes[(1, comps[c][3])]
            pred[c] = encode_block(bw, coeffs[c][y][x], pred[c], dc_codes, ac_codes, trailing_zrl)
    bw.pad(pad_bit)
    out += bw.take() + bytes(tail) + b"\xFF" * fill_bytes + b"\xFF\xD9"
    return bytes(out)


def scan_coefficients(width, height, comps, coeffs):
    """what a decoder reads back: every component's blocks as read_jpeg lays them out (components one after
    another, MCU-padded), the blocks a one-component scan does not cover zero -> one int64 vector"""
    n = len(comps)
    cols, rows, sizes = mcu_grid(width, height, comps)
    parts = []
    for c in range(n):
        a = np.zeros((sizes[c][1], sizes[c][0], 64), np.int64)
        if n == 1:
            bx, by = covered_blocks(width, height, comps, c)
            a[:by, :bx] = np.asarray(coeffs[c])[:by, :bx]
        else:
            a[:] = np.asarray(coeffs[c])
        parts.append(a.reshape(-1))
    return np.concatenate(parts)
