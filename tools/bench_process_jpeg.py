#!/usr/bin/env python
"""The encoder's JPEG input from host bytes (gb200_process_jpeg) against the same file held in CUDA memory
(gb200_process_jpeg_from_device), on Pillow-written q90 4:4:4 files of 1920x1080 and 4000x3000 from seeded
noise + gradient images, each with and without a restart marker every 4 MCUs.  Per file and entry (medians
over --rounds calls, the two entries alternating, after one untimed call of each on a small file):

  ms_wall          wall time of the call
  ms_device_setup  the call's own setup time: for the host entry from after read_jpeg to the resident
                   original; for the tensor entry from the call's start (header read, device decode) to it
  ms_total         the call's own total, measured from the same points
  h2d_bytes        bytes uploaded by the call
  d2h_bytes        bytes copied back by the call
  route            "device" where the tensor entry copied back less than the file, else "host"

and whether both entries gave the same bytes, with the card's name and power limit read in the same run
(nvidia-smi, read-only queries).  The host entry's ms_* start after read_jpeg, so ms_wall is the figure to
compare.  Prints one JSON line; --out also writes it to a file.  Without a GPU the script fails."""
import argparse
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import guetzli_b200 as gb  # noqa: E402
from guetzli_b200 import synth  # noqa: E402
from bench_image_inputs import gpu_info  # noqa: E402

SHAPES = {"1920x1080": (1080, 1920), "4000x3000": (3000, 4000)}
QUALITY = 90


def pillow_444(h, w, restart):
    from PIL import Image
    b = io.BytesIO()
    kw = {"restart_marker_blocks": restart} if restart else {}
    Image.fromarray(synth.gradnoise(h, w, 7)).save(b, "JPEG", quality=90, subsampling=0, **kw)
    return b.getvalue()


def call(lib, b, tensor):
    import torch
    src = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if tensor else b
    torch.cuda.synchronize()
    st = gb.ProcessStats()
    p = gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(QUALITY, lib=lib))
    t0 = time.perf_counter()
    ok, out = gb.process_jpeg(p, st, src, lib=lib)
    wall = 1e3 * (time.perf_counter() - t0)
    if not ok:
        raise RuntimeError(gb.last_error(lib=lib))
    d = st.device
    return out, {"ms_wall": wall, "ms_device_setup": d["ms_device_setup"], "ms_total": d["ms_total"],
                 "h2d_bytes": d["h2d_bytes"], "d2h_bytes": d["d2h_bytes"]}


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated subset of " + ",".join(SHAPES))
    ap.add_argument("--out")
    args = ap.parse_args()
    lib = gb.load_library()
    if lib.gb200_device_count() < 1:
        raise SystemExit("bench_process_jpeg: no CUDA device")
    small = pillow_444(64, 96, 0)
    call(lib, small, False)
    call(lib, small, True)
    res = {"gpu": gpu_info(0), "quality": QUALITY, "files": {}}
    for shape in args.shapes.split(","):
        h, w = SHAPES[shape]
        for restart in (0, 4):
            b = pillow_444(h, w, restart)
            runs = {"host": [], "device": []}
            outs = {}
            for _ in range(args.rounds):
                for entry, tensor in (("host", False), ("device", True)):
                    outs[entry], r = call(lib, b, tensor)
                    runs[entry].append(r)
            row = {"bytes": len(b), "same_output": outs["host"] == outs["device"]}
            for entry, rs in runs.items():
                row[entry] = {k: median([r[k] for r in rs]) for k in rs[0]}
            row["device"]["route"] = "device" if row["device"]["d2h_bytes"] - row["host"]["d2h_bytes"] < len(b) else "host"
            res["files"][f"{shape}_444_rst{restart}"] = row
            print(json.dumps({f"{shape}_444_rst{restart}": row}), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
