"""Synthetic sRGB inputs named by BASELINE.json / SURVEY.md §8(d).

numpy >= 2, PCG64 via np.random.default_rng(seed); every caller should log
sha256 of the returned bytes.
"""
import hashlib
import numpy as np


def noise(h, w, seed):
    """Uniform sRGB noise: rng.integers(0, 256, (H, W, 3), uint8)."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def gradnoise(h, w, seed, sigma=8.0):
    """Colour gradient plus Gaussian noise (sigma in 8-bit code values)."""
    rng = np.random.default_rng(seed)
    x = np.arange(w, dtype=np.float64)[None, :]
    y = np.arange(h, dtype=np.float64)[:, None]
    img = np.empty((h, w, 3), dtype=np.float64)
    img[..., 0] = x * 255.0 / (w - 1) + 0 * y
    img[..., 1] = y * 255.0 / (h - 1) + 0 * x
    img[..., 2] = (x + y) * 255.0 / (w + h - 2)
    img += rng.normal(0.0, sigma, (h, w, 3))
    return np.round(np.clip(img, 0.0, 255.0)).astype(np.uint8)


def sha256(arr):
    return hashlib.sha256(np.ascontiguousarray(arr).tobytes()).hexdigest()


def flat_blocks_gray(h, w, seed):
    """gradnoise turned gray, every 8x8 block shifted to a mean of 128: the AC content of noise with DC
    differences near 0 (jpeg_gray_as_444 regroups the DC chains, which would wander away otherwise)."""
    g = gradnoise(h, w, seed).astype(np.float64).mean(axis=2)
    hb, wb = (h + 7) // 8, (w + 7) // 8
    p = np.pad(g, ((0, 8 * hb - h), (0, 8 * wb - w)), mode="edge").reshape(hb, 8, wb, 8)
    p = p - p.mean(axis=(1, 3), keepdims=True) + 128.0
    return np.clip(np.round(p.reshape(8 * hb, 8 * wb)[:h, :w]), 0, 255).astype(np.uint8)


def jpeg_gray_as_444(gray_jpeg, w, h):
    """A 4:4:4 JPEG file whose three components share DHT tables 0 / 0 and quant table 0, as an encoder that
    clusters its histograms may write, made from a baseline gray file of 3 w x h (w a multiple of 8): its
    blocks in raster order are the 4:4:4 MCUs' blocks, so only the SOF, the SOS and the restart interval (a
    multiple of 3 gray blocks, to MCUs) are rewritten."""
    b, out, pos = gray_jpeg, bytearray(gray_jpeg[:2]), 2
    while True:
        marker, n = b[pos + 1], (b[pos + 2] << 8) | b[pos + 3]
        if marker == 0xc0:
            out += bytes([0xff, 0xc0, 0, 17, 8, h >> 8, h & 255, w >> 8, w & 255, 3,
                          1, 0x11, 0, 2, 0x11, 0, 3, 0x11, 0])
        elif marker == 0xdd:
            r = (b[pos + 4] << 8) | b[pos + 5]
            assert r % 3 == 0, "the gray restart interval must be a multiple of 3 blocks"
            out += bytes([0xff, 0xdd, 0, 4, (r // 3) >> 8, (r // 3) & 255])
        elif marker == 0xda:
            return bytes(out + bytes([0xff, 0xda, 0, 12, 3, 1, 0x00, 2, 0x00, 3, 0x00, 0, 63, 0]) + b[pos + 2 + n:])
        else:
            out += b[pos:pos + 2 + n]
        pos += 2 + n
