#!/usr/bin/env python
"""Where the time of gb.decode_jpeg goes, for calls of 1 and 64 files of three kinds: 768x512 q90 4:4:4,
768x512 q90 4:2:0 and 1920x1080 q90 4:2:0 (files written with Pillow from seeded noise + gradient images).
For each call it reports (medians over --rounds calls, after one untimed call):

  ms_call        wall time of decode_jpeg into CUDA tensors, up to torch.cuda.synchronize()
  ms_parse       host entropy decoding of the call's files (read_jpeg, through gb200_debug_read_jpeg, which
                 also copies the coefficients out)
  ms_device      the two decode kernels (jpeg_idct_islow, jpeg_upsample_ycc_rgb), CUDA events (gb200_profile)
  h2d_bytes      bytes uploaded by one call (coefficients and tables)
  ms_pillow      Pillow's decode plus torch upload of the same files, where Pillow is installed

and the card's name and power limit, read in the same run (nvidia-smi, read-only queries).  Prints one JSON
line; --out also writes it to a file.  There is no CPU mode: without a GPU the script fails."""
import argparse
import ctypes as C
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import guetzli_b200 as gb  # noqa: E402
from guetzli_b200 import synth  # noqa: E402
from bench_image_inputs import gpu_info  # noqa: E402

KINDS = {"768x512_444": (512, 768, 0), "768x512_420": (512, 768, 2), "1920x1080_420": (1080, 1920, 2)}


def jpeg_files(kind, n):
    from PIL import Image
    h, w, sub = KINDS[kind]
    out = []
    for i in range(min(n, 4)):  # four distinct files, repeated
        b = io.BytesIO()
        Image.fromarray(synth.gradnoise(h, w, 100 + i)).save(b, "JPEG", quality=90, subsampling=sub)
        out.append(b.getvalue())
    return [out[i % len(out)] for i in range(n)]


def profile(lib):
    names = (C.c_char * 48 * 256)()
    launches, ms, el = (C.c_long * 256)(), (C.c_double * 256)(), (C.c_double * 256)()
    n = lib.gb200_profile_get(names, launches, ms, el, 256)
    return {bytes(names[i]).split(b"\0")[0].decode(): ms[i] for i in range(n)}


def median(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    lib = gb.load_library()
    if lib.gb200_device_count() < 1:
        raise SystemExit("bench_jpeg_decode: no CUDA device")
    scratch = np.zeros(1 << 22, np.int16)
    dims = (C.c_int * 11)()
    res = {"calls": {}}
    for kind in KINDS:
        for n in (1, 64):
            files = jpeg_files(kind, n)
            gb.decode_jpeg(files)
            torch.cuda.synchronize()
            call, parse, dev, pil = [], [], [], []
            for _ in range(args.rounds):
                lib.gb200_profile_reset()
                lib.gb200_profile_enable(1)
                _, h0, _ = gb.counters(lib=lib)
                t0 = time.perf_counter()
                gb.decode_jpeg(files)
                torch.cuda.synchronize()
                call.append((time.perf_counter() - t0) * 1e3)
                _, h1, _ = gb.counters(lib=lib)
                lib.gb200_profile_enable(0)
                p = profile(lib)
                dev.append(p.get("jpeg_idct_islow", 0.0) + p.get("jpeg_upsample_ycc_rgb", 0.0))
                t0 = time.perf_counter()
                for f in files:
                    b = np.frombuffer(f, np.uint8)
                    lib.gb200_debug_read_jpeg(b.ctypes.data, b.size, dims, scratch.ctypes.data, scratch.size)
                parse.append((time.perf_counter() - t0) * 1e3)
                try:
                    from PIL import Image
                    t0 = time.perf_counter()
                    for f in files:
                        torch.from_numpy(np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))).cuda()
                    torch.cuda.synchronize()
                    pil.append((time.perf_counter() - t0) * 1e3)
                except ImportError:
                    pass
            res["calls"][f"{kind}_x{n}"] = {
                "ms_call": round(median(call), 3), "ms_parse": round(median(parse), 3),
                "ms_device": round(median(dev), 3), "h2d_bytes": h1 - h0,
                "ms_pillow": round(median(pil), 3) if pil else None}
    res.update(gpu_info(0))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
