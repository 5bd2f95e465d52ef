#!/usr/bin/env python
"""Device set-up time of one encode (ms_device_setup: the image context made, the image uploaded or read in
place and converted, up to the start of the search) for one RGB image (default 1920x1080), two ways:

  host   gb.process on a numpy array: the RGB bytes cross PCIe into the context
  cuda   gb.process_image on a CUDA torch tensor: the context reads the tensor in place (ingest_u8)

The modes alternate for --rounds rounds after one untimed call each; the result has every round's time, the
bytes each call uploaded, whether the two JPEGs are equal, and the card's name and power limit, read in the
same run (nvidia-smi, read-only queries).  Prints one JSON line; --out also writes it to a file.  There is no
CPU mode: without a GPU the script fails."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import guetzli_b200 as gb  # noqa: E402
from guetzli_b200 import synth  # noqa: E402


def gpu_info(device):
    q = "name,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=" + q, "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--quality", type=float, default=95)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    lib = gb.load_library()
    if lib.gb200_device_count() < 1:
        raise SystemExit("bench_image_inputs: no CUDA device")
    rgb = synth.noise(args.h, args.w, 1234)
    t = torch.from_numpy(rgb).cuda()
    torch.cuda.synchronize()
    p = gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(args.quality))

    def host():
        st = gb.ProcessStats()
        return gb.process(p, st, rgb, args.w, args.h), st

    def cuda():
        st = gb.ProcessStats()
        return gb.process_image(p, st, t), st

    modes = {"host": host, "cuda": cuda}
    ms = {k: [] for k in modes}
    h2d, jpeg = {}, {}
    for k, f in modes.items():
        f()  # untimed
    for _ in range(args.rounds):
        for k, f in modes.items():
            (ok, data), st = f()
            assert ok, k
            ms[k].append(round(st.device["ms_device_setup"], 3))
            h2d[k], jpeg[k] = st.device["h2d_bytes"], data
    res = {"image": f"{args.w}x{args.h}", "ms_device_setup": ms,
           "ms_device_setup_median": {k: sorted(v)[len(v) // 2] for k, v in ms.items()},
           "h2d_bytes": h2d, "jpeg_equal": jpeg["host"] == jpeg["cuda"]}
    res.update(gpu_info(0))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
