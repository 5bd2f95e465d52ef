#!/usr/bin/env python3
"""What libjpeg-turbo (through Pillow, with its default SIMD) decodes from JPEG files, recorded for
tests/test_jpeg_decode.py: -> tests/golden/jpeg_decode_reference_answers.json (sha256 of each decode,
or the refusal the file should meet) and tests/golden/jpeg_decode_files.npz (the generated files and
the pixels of the small ones).  Runs where Pillow is installed; the tests read only what it writes.

Generated files:
  sweep_<sub>_<w>x<h>: Pillow-written q90 files, <sub> in 444, 422, 420, gray, at every width 1..24, 33,
      47, 65 with height 9, every height with width 11, and every square size;
  rgb_ids: base444_q90 without its JFIF APP0 and with component ids 'R', 'G', 'B' (an RGB file);
  q255_dc: gb.write_jpeg at q = 255 with DC-only blocks of quantised DC up to 128 in magnitude (the
      largest it emits), whose outputs wrap through libjpeg's range-limit table;
  q255_ac: the same with random AC coefficients up to 128, where libjpeg-turbo's SIMD IDCT leaves
      its C IDCT (refused);
  sub440, sub411: 4:2:2 and 4:2:0 files whose luma sampling was edited to 1x2 and 4x1, with the frame
      size swapped so that the scan data still matches;
  prog_cut: prog444_q85 without its last two scans (coefficients not refined to bit 0);
  guetzli_q90: what the encoder (the CPU port, bit for bit the reference) makes of the smoke test's
      64x96 image at quality 90.
Pixels are kept for the generated files and for jpeg/sub420.
"""
import hashlib
import io
import json
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from guetzli_b200 import synth  # noqa: E402

SIZES = list(range(1, 25)) + [33, 47, 65]
SUBS = {"444": 0, "422": 1, "420": 2, "gray": None}


def pil_jpeg(rgb, sub, **kw):
    b = io.BytesIO()
    im = Image.fromarray(rgb)
    if sub is None:
        im.convert("L").save(b, "JPEG", quality=90, **kw)
    else:
        im.save(b, "JPEG", quality=90, subsampling=sub, **kw)
    return b.getvalue()


def pil_decode(data):
    im = Image.open(io.BytesIO(data))
    im.load()
    return np.asarray(im.convert("RGB") if im.mode == "L" else im)


def segments(data):
    """(marker, start, end) of the segments before the first SOS, and the position of every SOS."""
    pos, segs, sos = 2, [], []
    while pos + 4 <= len(data):
        m = data[pos + 1]
        ln = (data[pos + 2] << 8) | data[pos + 3]
        segs.append((m, pos, pos + 2 + ln))
        if m == 0xDA:
            break
        pos += 2 + ln
    i = 0
    while True:
        i = data.find(b"\xff\xda", i)
        if i < 0:
            return segs, sos
        sos.append(i)
        i += 2


def edit_sof(data, sampling0, w, h):
    segs, _ = segments(data)
    b = bytearray(data)
    for m, s, _e in segs:
        if m in (0xC0, 0xC2):
            b[s + 5:s + 7] = h.to_bytes(2, "big")
            b[s + 7:s + 9] = w.to_bytes(2, "big")
            b[s + 11] = sampling0
    return bytes(b)


def rgb_ids(data):
    segs, _ = segments(data)
    b = bytearray()
    b += data[:2]
    last = 2
    for m, s, e in segs:
        if m == 0xE0:
            b += data[last:s]
            last = e
    b += data[last:]
    for m, s, _e in segments(bytes(b))[0]:
        if m == 0xC0:
            for k, cid in enumerate(b"RGB"):
                b[s + 10 + 3 * k] = cid
        if m == 0xDA:
            for k, cid in enumerate(b"RGB"):
                b[s + 5 + 2 * k] = cid
    return bytes(b)


def write_jpeg_q255(ac):
    import guetzli_b200 as gb
    rng = np.random.default_rng(7)
    w, h = 64, 40
    nb = (w // 8) * (h // 8)
    c = np.zeros((3, nb, 64), np.int32)
    # quantised DC values whose 4 x 255 x DC, wrapped to 16 bits as libjpeg-turbo's SIMD DC shortcut
    # wraps it, still descales into [-512, 511]: there its SIMD and C IDCTs agree, and for |DC| > 16 the
    # C IDCT's output leaves [-512, 511] and wraps through the range-limit table
    ok = [v for v in range(-128, 129) if -512 <= ((((1020 * v + 32768) % 65536) - 32768) + 16) >> 5 <= 511]
    c[:, :, 0] = np.resize(np.array(ok, np.int32), 3 * nb).reshape(3, nb)
    if ac:
        c[:, :, 1:] = rng.integers(-128, 129, size=(3, nb, 63))
    return gb.write_jpeg(np.clip(c * 255, -32768, 32767), w, h, np.full(192, 255))


def generated():
    files = {}
    for name, sub in SUBS.items():
        for w, h in sorted({(s, 9) for s in SIZES} | {(11, s) for s in SIZES} | {(s, s) for s in SIZES}):
            rgb = np.random.default_rng(w * 100 + h).integers(0, 256, size=(h, w, 3), dtype=np.uint8)
            files[f"sweep_{name}_{w}x{h}"] = pil_jpeg(rgb, sub)
    base = open(os.path.join(HERE, "jpeg", "base444_q90.jpg"), "rb").read()
    files["rgb_ids"] = rgb_ids(base)
    files["q255_dc"] = write_jpeg_q255(False)
    files["q255_ac"] = write_jpeg_q255(True)
    files["sub440"] = edit_sof(pil_jpeg(synth.gradnoise(16, 32, 1), 1), 0x12, 16, 32)
    files["sub411"] = edit_sof(pil_jpeg(synth.gradnoise(32, 32, 2), 2), 0x41, 64, 16)
    prog = open(os.path.join(HERE, "jpeg", "prog444_q85.jpg"), "rb").read()
    cut = segments(prog)[1][-2]
    files["prog_cut"] = prog[:cut] + b"\xff\xd9"
    import guetzli_b200 as gb
    port = gb.load_library(os.path.join(HERE, "..", "..", "oracle", "_build", "libguetzli_port.so"))
    params = gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(90, lib=port))
    ok, files["guetzli_q90"] = gb.process(params, None, synth.gradnoise(64, 96, 7), 96, 64, lib=port)
    assert ok
    return files


def main():
    answers, arrays = {}, {}
    fixtures = sorted(f[:-4] for f in os.listdir(os.path.join(HERE, "jpeg")) if f.endswith(".jpg"))
    items = [("jpeg/" + f, open(os.path.join(HERE, "jpeg", f + ".jpg"), "rb").read()) for f in fixtures]
    items += sorted(generated().items())
    for name, data in items:
        if not name.startswith("jpeg/"):
            arrays["file_" + name] = np.frombuffer(data, np.uint8)
        try:
            px = pil_decode(data)
        except Exception as e:  # noqa: BLE001
            answers[name] = {"pillow": "error: " + str(e)}
            continue
        answers[name] = {"pillow": hashlib.sha256(np.ascontiguousarray(px).tobytes()).hexdigest(),
                         "shape": list(px.shape)}
        if (not name.startswith("jpeg/") or name == "jpeg/sub420") and px.ndim == 3 and px.shape[2] == 3:
            arrays["px_" + name.replace("/", "_")] = px
    import PIL.features
    meta = {"pillow": PIL.__version__ if hasattr(PIL, "__version__") else "",
            "libjpeg": PIL.features.version("jpg"), "libjpeg_turbo": bool(PIL.features.check_feature("libjpeg_turbo"))}
    json.dump({"meta": meta, "files": answers}, open(os.path.join(HERE, "jpeg_decode_reference_answers.json"), "w"),
              indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, "jpeg_decode_files.npz"), **arrays)
    print(len(answers), "answers")


if __name__ == "__main__":
    import PIL  # noqa: F401
    main()
