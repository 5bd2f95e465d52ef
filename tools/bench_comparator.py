#!/usr/bin/env python
"""Wall time per scored image of the stand-alone butteraugli, three ways, at one size (default 1920x1080):

  pairwise        one gb200_butteraugli_diffmap per pair: a context is built, the original is
                  analysed, both images cross PCIe, the pair is scored, everything is freed
  comparator_host one resident gb200_butteraugli_comparator, candidates and diffmaps in host memory
  comparator_cuda the same comparator, candidates and diffmaps as CUDA torch tensors

Every call returns once its diffmap is written, so a host clock around `--n` calls is the time of
the work.  The modes run in turn for `--rounds` rounds (the spread between rounds is part of the
result), after `--warmup` untimed calls each.  The card's name and power limit are read in the
same run (nvidia-smi, read-only queries).  Prints one JSON line; --out also writes it to a file.
There is no CPU mode: without a GPU the script fails."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

import guetzli_b200 as gb  # noqa: E402
from guetzli_b200 import synth  # noqa: E402


def linear(rgb):
    """sRGB bytes [h][w][3] -> planar linear RGB float32 [3][h][w] in 0..255."""
    v = rgb.astype(np.float64) / 255.0
    lin = np.where(v <= 0.04045, v / 12.92, ((v + 0.055) / 1.055) ** 2.4) * 255.0
    return np.ascontiguousarray(lin.transpose(2, 0, 1)).astype(np.float32)


def gpu_info(device):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=" + q, "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        return {"gpu": None, "power_limit": None, "sm_max_clock": None, "nvidia_smi_error": str(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--n", type=int, default=20, help="timed calls per mode and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    lib = gb.load_library()
    if lib.gb200_device_count() < 1:
        raise SystemExit("bench_comparator: no CUDA device; the product has no CPU fallback")
    import torch
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)

    h, w = args.h, args.w
    base = synth.gradnoise(h, w, 11).astype(int)
    orig = linear(base.astype(np.uint8))
    cands = [linear(np.clip(base + synth.noise(h, w, 200 + k) % 7 - 3, 0, 255).astype(np.uint8)) for k in range(args.n)]
    cands_dev = [torch.from_numpy(c).to(dev) for c in cands]
    torch.cuda.synchronize(dev)
    cmp = gb.Comparator(orig, device=args.device)

    def pairwise(i):
        return gb.api.butteraugli_diffmap(orig, cands[i], device=args.device)[1]

    def comparator_host(i):
        return cmp.diffmap(cands[i])[1]

    def comparator_cuda(i):
        return cmp.diffmap(cands_dev[i])[1]

    modes = {"pairwise": pairwise, "comparator_host": comparator_host, "comparator_cuda": comparator_cuda}
    scores = {}
    for name, f in modes.items():
        for i in range(args.warmup):
            f(i % args.n)
        scores[name] = [f(i) for i in range(args.n)]
    identical = all(scores[m] == scores["pairwise"] for m in modes)

    ms = {m: [] for m in modes}
    for _ in range(args.rounds):
        for name, f in modes.items():
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for i in range(args.n):
                f(i)
            torch.cuda.synchronize(dev)
            ms[name].append((time.perf_counter() - t0) / args.n * 1e3)
    cmp.close()

    result = {"size": f"{w}x{h}", "calls_per_round": args.n, "rounds": args.rounds,
              "ms_per_image": {m: {"median": round(statistics.median(v), 3), "min": round(min(v), 3),
                                   "max": round(max(v), 3)} for m, v in ms.items()},
              "scores_identical_across_modes": identical}
    result.update(gpu_info(args.device))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
