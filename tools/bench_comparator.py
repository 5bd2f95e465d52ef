#!/usr/bin/env python
"""Wall time per scored image of the stand-alone butteraugli, three ways, at one size (default 1920x1080):

  pairwise        one gb200_butteraugli_diffmap per pair: a context is built, the original is
                  analysed, both images cross PCIe, the pair is scored, everything is freed
  comparator_host one resident gb200_butteraugli_comparator, candidates and diffmaps in host memory
  comparator_cuda the same comparator, candidates and diffmaps as CUDA torch tensors

With --batch N, two more modes score N distinct pairs (a different original in each) per call:

  batch_cuda      one gb200_butteraugli_batch of capacity N, pairs and diffmaps as CUDA torch tensors
  batch_host      the same batch, pairs and diffmaps in host memory

and two more score N distinct candidates against the one original per call:

  comparator_batch_cuda  one comparator of capacity N, candidates and diffmaps as CUDA torch tensors
  comparator_batch_host  the same comparator, candidates and diffmaps in host memory

and four more take the same images as 8-bit sRGB (RGB, 3 bytes per pixel), converted on the device:

  batch_srgb_cuda, batch_srgb_host                       ButteraugliBatch.diffmap_srgb
  comparator_batch_srgb_cuda, comparator_batch_srgb_host  a comparator made by Comparator.from_srgb

Their scores must equal their float twins' (scores_srgb_equal_float).

With --sizes, pairs of different sizes are scored in sets (SIZE_SETS; "uniform" is a same-size set, for the
mixed-size entry against the same-size one), ms per set, four or five ways:

  sizes_cuda      one ButteraugliBatch (the set's largest width x height) and diffmap_sizes, CUDA tensors
  sizes_host      the same with numpy arrays
  grouped_cuda    one ButteraugliBatch per distinct size (made before timing), one diffmap call per size:
                  the best a caller can do without diffmap_sizes
  pairwise        one Comparator per pair, made, scored once and closed: scoring the pairs one by one
  batch_cuda      ("uniform" only) the same-size entry on the same pairs

and each float mode of the mixed-size entry is followed by its 8-bit twin on the same images as RGB bytes:

  sizes_srgb_cuda ButteraugliBatch.diffmap_sizes_srgb, uint8 CUDA tensors
  sizes_srgb_host the same with numpy arrays

The set "kodak_rgba" has Kodak-like shapes with alpha on half the pairs.  Its float modes score the pairs
over black and the RGBA pairs over white as well, and keep the larger score (black on a tie), as the 8-bit
entry does; grouping and pairwise scoring are not timed there.  Per set, the result reports whether the
8-bit scores equal the float scores (scores_srgb_equal_float) and the device memory the batch holds after
creation and what its first 8-bit mixed call adds.

A set larger than what one batch's arena holds goes in calls of --sizes-capacity pairs.  The result gains ms per pair or
candidate of the batched modes, MPix/s (scored pixels per second) of every mode, and the device memory
the batch and the batched comparators (RGB, and RGBA with its two originals) hold after creation and after
their first 8-bit call (MiB, from torch.cuda.mem_get_info after gb200_trim_memory).  Every call returns once its diffmaps are written, so a host clock around `--n` calls is the
time of the work.  The modes run in turn for `--rounds` rounds (the spread between rounds is part of the
result), after `--warmup` untimed calls each.  The card's name and power limit are read in the
same run (nvidia-smi, read-only queries).  Prints one JSON line; --out also writes it to a file.
There is no CPU mode: without a GPU the script fails.

With --set, two rate-distortion sweeps (SET_WORKLOADS: K originals of sizes of their own, Q candidates
each) are scored in calls of --sizes-capacity candidates, ms per candidate, in modes that alternate in
every round:

  set_cuda          one ComparatorSet of all K originals (made before timing), CUDA tensors
  set_host          the same set, numpy arrays
  sizes_cuda        the same pairs through ButteraugliBatch.diffmap_sizes, CUDA tensors: every call
                    analyses and uploads its originals again
  sizes_host        the same with numpy arrays
  comparators_cuda  ("kodak" only) one Comparator of capacity Q per original, made before timing, one call
                    per original

It reports the device memory each holds after gb200_trim_memory, the bytes each host mode uploads per
candidate, and whether every mode's scores are equal."""
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
    ap.add_argument("--batch", type=int, default=0, help="pairs per call of the batch modes (0: no batch modes)")
    ap.add_argument("--sizes", action="store_true", help="also time the mixed-size sets (SIZE_SETS)")
    ap.add_argument("--sizes-only", action="store_true", help="time the mixed-size sets and nothing else")
    ap.add_argument("--sizes-capacity", type=int, default=64,
                    help="pairs per call of a set whose largest size is 1920x1080 (the arena of 256 such slots "
                         "does not fit in 80 GB)")
    ap.add_argument("--set", action="store_true", help="time the comparator-set sweeps and nothing else")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    lib = gb.load_library()
    if lib.gb200_device_count() < 1:
        raise SystemExit("bench_comparator: no CUDA device; the product has no CPU fallback")
    import torch
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)

    if args.set:
        result = {"set": bench_set(args, dev, torch)}
        result.update(gpu_info(args.device))
        emit(result, args.out)
        return
    if args.sizes_only:
        result = {"sizes": bench_sizes(args, dev, torch)}
        result.update(gpu_info(args.device))
        emit(result, args.out)
        return
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
    per_call = {m: 1 for m in modes}
    memory = {}
    if args.batch > 0:
        nb = args.batch
        u0 = np.stack([synth.gradnoise(h, w, 1000 + i) for i in range(nb)])
        u1 = np.stack([np.clip(synth.gradnoise(h, w, 1000 + i).astype(int) + synth.noise(h, w, 3000 + i) % 7 - 3,
                               0, 255).astype(np.uint8) for i in range(nb)])
        b0 = np.stack([linear(x) for x in u0])
        b1 = np.stack([linear(x) for x in u1])
        b0_dev, b1_dev = torch.from_numpy(b0).to(dev), torch.from_numpy(b1).to(dev)
        u0_dev, u1_dev = torch.from_numpy(u0).to(dev), torch.from_numpy(u1).to(dev)
        uc = np.stack([np.clip(base + synth.noise(h, w, 5000 + k) % 7 - 3, 0, 255).astype(np.uint8) for k in range(nb)])
        c1 = np.stack([linear(x) for x in uc])
        c1_dev, uc_dev = torch.from_numpy(c1).to(dev), torch.from_numpy(uc).to(dev)
        torch.cuda.synchronize(dev)

        def free_mib():
            lib.gb200_trim_memory()
            torch.cuda.synchronize(dev)
            return torch.cuda.mem_get_info(dev)[0] / 2**20

        f0 = free_mib()
        batch = gb.ButteraugliBatch(h, w, nb, device=args.device)
        f1 = free_mib()
        batch.diffmap_srgb(u0, u1)
        f2 = free_mib()
        cmpb = gb.Comparator(orig, device=args.device, capacity=nb)
        f3 = free_mib()
        cmps = gb.Comparator.from_srgb(base.astype(np.uint8), device=args.device, capacity=nb)
        f4 = free_mib()
        cmps.diffmap(uc)
        f5 = free_mib()
        # an RGBA comparator (two resident originals), measured and freed again before the timed modes
        alpha = (synth.noise(h, w, 77)[..., :1] | 1).astype(np.uint8)
        cmpa = gb.Comparator.from_srgb(np.concatenate([base.astype(np.uint8), alpha], axis=2), device=args.device,
                                       capacity=nb)
        f6 = free_mib()
        cmpa.diffmap(np.concatenate([uc, np.broadcast_to(alpha, uc.shape[:3] + (1,))], axis=3))
        f7 = free_mib()
        cmpa.close()
        memory = {"batch_mib": round(f0 - f1, 1), "batch_srgb_buffers_mib": round(f1 - f2, 1),
                  "comparator_batch_mib": round(f2 - f3, 1), "comparator_batch_srgb_mib": round(f3 - f4, 1),
                  "comparator_batch_srgb_buffers_mib": round(f4 - f5, 1),
                  "comparator_batch_srgba_mib": round(f5 - f6, 1),
                  "comparator_batch_srgba_buffers_mib": round(f6 - f7, 1)}

        def batch_srgb_cuda(i):
            return batch.diffmap_srgb(u0_dev, u1_dev)[1].tolist()

        def batch_srgb_host(i):
            return batch.diffmap_srgb(u0, u1)[1].tolist()

        def comparator_batch_srgb_cuda(i):
            return cmps.diffmap(uc_dev)[1].tolist()

        def comparator_batch_srgb_host(i):
            return cmps.diffmap(uc)[1].tolist()

        def comparator_batch_cuda(i):
            return cmpb.diffmap(c1_dev)[1].tolist()

        def comparator_batch_host(i):
            return cmpb.diffmap(c1)[1].tolist()

        def batch_cuda(i):
            return batch.diffmap(b0_dev, b1_dev)[1].tolist()

        def batch_host(i):
            return batch.diffmap(b0, b1)[1].tolist()

        # each 8-bit mode right after its float twin
        modes.update(batch_cuda=batch_cuda, batch_srgb_cuda=batch_srgb_cuda, batch_host=batch_host,
                     batch_srgb_host=batch_srgb_host, comparator_batch_cuda=comparator_batch_cuda,
                     comparator_batch_srgb_cuda=comparator_batch_srgb_cuda, comparator_batch_host=comparator_batch_host,
                     comparator_batch_srgb_host=comparator_batch_srgb_host)
        per_call.update({m: nb for m in modes if "batch" in m})
    scores = {}
    for name, f in modes.items():
        for i in range(args.warmup):
            f(i % args.n)
        scores[name] = [f(i) for i in range(args.n)]
    single = ["pairwise", "comparator_host", "comparator_cuda"]
    identical = all(scores[m] == scores["pairwise"] for m in single)

    ms = {m: [] for m in modes}
    for _ in range(args.rounds):
        for name, f in modes.items():
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for i in range(args.n):
                f(i)
            torch.cuda.synchronize(dev)
            ms[name].append((time.perf_counter() - t0) / args.n * 1e3 / per_call[name])
    if args.batch > 0:
        # the last candidate of the batched comparator scores as it does alone
        cand_alone = cmp.diffmap(c1[-1])[1]
        cmpb.close()
        cmps.close()
    cmp.close()

    def stats(v):
        return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}

    result = {"size": f"{w}x{h}", "calls_per_round": args.n, "rounds": args.rounds,
              "ms_per_image": {m: stats(ms[m]) for m in single},
              "scores_identical_across_modes": identical}
    if args.batch > 0:
        batch.close()
        # every batch call scores the same pairs: host and device entry agree, and pair 0 scores as it
        # does alone
        alone = gb.api.butteraugli_diffmap(b0[0], b1[0], device=args.device)[1]
        result["batch"] = args.batch
        result["ms_per_pair"] = {m: stats(ms[m]) for m in ms if m.startswith("batch")}
        result["ms_per_candidate"] = {m: stats(ms[m]) for m in ms if m.startswith("comparator_batch")}
        result["mpix_per_s"] = {m: round(w * h / 1e3 / statistics.median(v), 2) for m, v in ms.items()}
        result["batch_scores_consistent"] = (all(s == scores["batch_cuda"][0] for m in ("batch_cuda", "batch_host")
                                                 for s in scores[m]) and scores["batch_cuda"][0][0] == alone)
        cb = ("comparator_batch_cuda", "comparator_batch_host")
        result["comparator_batch_scores_consistent"] = (
            all(s == scores[cb[0]][0] for m in cb for s in scores[m]) and scores[cb[0]][0][-1] == cand_alone)
        # the 8-bit modes score the converted planes of the float modes' images
        result["scores_srgb_equal_float"] = all(scores[m] == scores[m.replace("_srgb", "")] for m in ms if "_srgb" in m)
        result["device_memory"] = memory
    if args.sizes:
        result["sizes"] = bench_sizes(args, dev, torch)
    result.update(gpu_info(args.device))
    emit(result, args.out)


def emit(result, out):
    line = json.dumps(result)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")


def over(img, bg):
    """uint8 [h][w][4] laid over the background bg in sRGB space, in integers, as the butteraugli tool does
    (butteraugli_main.cc:264-275) -> [h][w][3]; [h][w][3] as it is."""
    if img.shape[2] == 3:
        return img
    rgb, al = img[..., :3].astype(int), img[..., 3:].astype(int)
    v = (rgb * al + bg * (255 - al) + 127) // 255
    return np.where(al == 255, rgb, np.where(al == 0, bg, v)).astype(np.uint8)


def size_sets():
    """name -> [(h, w) of each pair]"""
    rng = np.random.default_rng(17)
    return {
        # Kodak-like: landscape and portrait 768x512 images mixed
        "kodak": [(512, 768) if i % 3 else (768, 512) for i in range(24)],
        # 256 pairs of random sizes from 32 to 256
        "random": [(int(a), int(b)) for a, b in rng.integers(32, 257, size=(256, 2))],
        # one 1920x1080 pair and 255 pairs of 64x64
        "hd_small": [(1080, 1920)] + [(64, 64)] * 255,
        # a same-size set: the mixed-size entry against the same-size one
        "uniform": [(256, 256)] * 64,
        # the Kodak-like shapes with alpha on every other pair
        "kodak_rgba": [(512, 768) if i % 3 else (768, 512) for i in range(24)],
    }


def bench_sizes(args, dev, torch):
    out = {}
    for name, shapes in size_sets().items():
        n = len(shapes)
        bh, bw = max(s[0] for s in shapes), max(s[1] for s in shapes)
        cap = min(n, args.sizes_capacity) if bh * bw >= 1920 * 1080 else n
        alpha = name.endswith("_rgba")
        u0, u1 = [], []  # the 8-bit images
        for i, (h, w) in enumerate(shapes):
            u = synth.gradnoise(h, w, 100 + i).astype(int)
            v = np.clip(u + synth.noise(h, w, 900 + i) % 7 - 3, 0, 255).astype(np.uint8)
            u = u.astype(np.uint8)
            if alpha and i % 2:  # every alpha value; the candidate's alpha as the original's
                al = (synth.noise(h, w, 500 + i)[..., :1].astype(int) * 37 % 256).astype(np.uint8)
                u, v = np.concatenate([u, al], axis=2), np.concatenate([v, al], axis=2)
            u0.append(u)
            u1.append(v)
        rgba = [i for i in range(n) if u0[i].shape[2] == 4]
        # the float images: the pairs over black, and the RGBA pairs over white
        a, b = [linear(over(x, 0)) for x in u0], [linear(over(x, 0)) for x in u1]
        aw, bw_ = [linear(over(u0[i], 255)) for i in rgba], [linear(over(u1[i], 255)) for i in rgba]
        a_dev = [torch.from_numpy(x).to(dev) for x in a]
        b_dev = [torch.from_numpy(x).to(dev) for x in b]
        aw_dev = [torch.from_numpy(x).to(dev) for x in aw]
        bw_dev = [torch.from_numpy(x).to(dev) for x in bw_]
        u0_dev = [torch.from_numpy(x).to(dev) for x in u0]
        u1_dev = [torch.from_numpy(x).to(dev) for x in u1]
        torch.cuda.synchronize(dev)

        def free_mib():
            gb.load_library().gb200_trim_memory()
            torch.cuda.synchronize(dev)
            return torch.cuda.mem_get_info(dev)[0] / 2**20

        f0 = free_mib()
        batch = gb.ButteraugliBatch(bh, bw, cap, device=args.device)
        f1 = free_mib()
        batch.diffmap_sizes_srgb(u0[:cap], u1[:cap])
        f2 = free_mib()
        groups = {}
        for i, s in enumerate(shapes):
            groups.setdefault(s, []).append(i)
        timed_groups = {} if alpha else groups  # the RGBA set times no grouping
        per_size = {s: gb.ButteraugliBatch(s[0], s[1], len(ix), device=args.device) for s, ix in timed_groups.items()}
        stacked = {s: (torch.stack([a_dev[i] for i in ix]), torch.stack([b_dev[i] for i in ix]))
                   for s, ix in timed_groups.items()}
        torch.cuda.synchronize(dev)

        def in_calls(f, x, y):
            scores = []
            for k in range(0, len(x), cap):
                scores += f(x[k:k + cap], y[k:k + cap])[1].tolist()
            return scores

        def with_white(x, y, xw, yw):
            """the float scores over black, and for the RGBA pairs the larger one (black on a tie)"""
            scores = in_calls(batch.diffmap_sizes, x, y)
            if rgba:
                for i, v in zip(rgba, in_calls(batch.diffmap_sizes, xw, yw)):
                    scores[i] = v if v > scores[i] else scores[i]
            return scores

        def sizes_cuda():
            return with_white(a_dev, b_dev, aw_dev, bw_dev)

        def sizes_srgb_cuda():
            return in_calls(batch.diffmap_sizes_srgb, u0_dev, u1_dev)

        def sizes_host():
            return with_white(a, b, aw, bw_)

        def sizes_srgb_host():
            return in_calls(batch.diffmap_sizes_srgb, u0, u1)

        def grouped_cuda():
            scores = [0.0] * n
            for s, ix in groups.items():
                for i, v in zip(ix, per_size[s].diffmap(*stacked[s])[1].tolist()):
                    scores[i] = v
            return scores

        def pairwise():
            scores = []
            for i in range(n):
                c = gb.Comparator(a[i], device=args.device)
                scores.append(c.diffmap(b[i])[1])
                c.close()
            return scores

        modes = {"sizes_cuda": sizes_cuda, "sizes_srgb_cuda": sizes_srgb_cuda, "sizes_host": sizes_host,
                 "sizes_srgb_host": sizes_srgb_host, "grouped_cuda": grouped_cuda, "pairwise": pairwise}
        if alpha:
            del modes["grouped_cuda"], modes["pairwise"]
        elif len(groups) == 1:
            modes["batch_cuda"] = grouped_cuda  # one size: grouping is the same-size entry on all pairs
            del modes["grouped_cuda"]
        scores = {m: f() for m, f in modes.items()}  # also the warm-up
        ms = {m: [] for m in modes}
        for _ in range(args.rounds):
            for m, f in modes.items():
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize(dev)
                ms[m].append((time.perf_counter() - t0) * 1e3)
        batch.close()
        for x in per_size.values():
            x.close()
        mpix = sum(h * w for h, w in shapes) / 1e6
        out[name] = {"pairs": n, "distinct_sizes": len(groups), "batch": f"{bw}x{bh}", "capacity": cap,
                     "mpix": round(mpix, 3),
                     "ms_per_set": {m: {"median": round(statistics.median(v), 3), "min": round(min(v), 3),
                                        "max": round(max(v), 3)} for m, v in ms.items()},
                     "mpix_per_s": {m: round(mpix * 1e3 / statistics.median(v), 1) for m, v in ms.items()},
                     "scores_identical": all(v == scores["sizes_cuda"] for m, v in scores.items() if "_srgb" not in m),
                     "scores_srgb_equal_float": all(v == scores[m.replace("_srgb", "")] for m, v in scores.items()
                                                    if "_srgb" in m),
                     "rgba_pairs": len(rgba),
                     "device_memory": {"batch_mib": round(f0 - f1, 1), "sizes_srgb_buffers_mib": round(f1 - f2, 1)}}
    return out


def set_workloads():
    """name -> ([(h, w) of each original], candidates per original)"""
    rng = np.random.default_rng(23)
    return {
        # Kodak-like: 24 landscape and portrait 768x512 images, 8 quality settings each
        "kodak": ([(512, 768) if i % 3 else (768, 512) for i in range(24)], 8),
        # a folder of thumbnails: 1024 images of random sizes from 32 to 256, 4 quality settings each
        "thumbnails": ([(int(a), int(b)) for a, b in rng.integers(32, 257, size=(1024, 2))], 4),
    }


def bench_set(args, dev, torch):
    lib = gb.load_library()
    out = {}
    for name, (shapes, q) in set_workloads().items():
        k = len(shapes)
        cap = args.sizes_capacity
        u0 = [synth.gradnoise(h, w, 100 + i).astype(int) for i, (h, w) in enumerate(shapes)]
        orig = [linear(x.astype(np.uint8)) for x in u0]
        index = [i for i in range(k) for _ in range(q)]  # the candidates of an original are consecutive
        cands = [linear(np.clip(u0[i] + synth.noise(*shapes[i], 900 + j) % (3 + 2 * (j % q)) - (1 + j % q), 0, 255)
                        .astype(np.uint8)) for j, i in enumerate(index)]
        orig_dev = [torch.from_numpy(x).to(dev) for x in orig]
        cands_dev = [torch.from_numpy(x).to(dev) for x in cands]
        torch.cuda.synchronize(dev)
        n = len(index)
        bh, bw = max(s[0] for s in shapes), max(s[1] for s in shapes)

        def free_mib():
            lib.gb200_trim_memory()
            torch.cuda.synchronize(dev)
            return torch.cuda.mem_get_info(dev)[0] / 2**20

        memory = {}
        f0 = free_mib()
        cset = gb.ComparatorSet(orig, capacity=cap, device=args.device)
        memory["set_mib"] = round(f0 - free_mib(), 1)
        f0 = free_mib()
        batch = gb.ButteraugliBatch(bh, bw, cap, device=args.device)
        memory["sizes_batch_mib"] = round(f0 - free_mib(), 1)
        cmps = None
        if name == "kodak":
            f0 = free_mib()
            cmps = [gb.Comparator(x, device=args.device, capacity=q) for x in orig]
            memory["comparators_mib"] = round(f0 - free_mib(), 1)
            stacked = [torch.stack(cands_dev[i * q:(i + 1) * q]) for i in range(k)]
            torch.cuda.synchronize(dev)

        def in_calls(f, a, b):
            scores = []
            for j in range(0, n, cap):
                scores += f(a[j:j + cap], b[j:j + cap])[1].tolist()
            return scores

        def set_cuda():
            return in_calls(cset.diffmap, index, cands_dev)

        def set_host():
            return in_calls(cset.diffmap, index, cands)

        def sizes_cuda():
            return in_calls(batch.diffmap_sizes, [orig_dev[i] for i in index], cands_dev)

        def sizes_host():
            return in_calls(batch.diffmap_sizes, [orig[i] for i in index], cands)

        def comparators_cuda():
            return [v for i in range(k) for v in cmps[i].diffmap(stacked[i])[1].tolist()]

        modes = {"set_cuda": set_cuda, "set_host": set_host, "sizes_cuda": sizes_cuda, "sizes_host": sizes_host}
        if cmps is not None:
            modes["comparators_cuda"] = comparators_cuda
        scores, h2d = {}, {}
        for m, f in modes.items():  # also the warm-up
            before = gb.counters()[1]
            scores[m] = f()
            h2d[m] = (gb.counters()[1] - before) / n
        ms = {m: [] for m in modes}
        for _ in range(args.rounds):
            for m, f in modes.items():
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize(dev)
                ms[m].append((time.perf_counter() - t0) * 1e3 / n)
        cset.close()
        batch.close()
        for c in cmps or []:
            c.close()
        out[name] = {"originals": k, "candidates_per_original": q, "candidates": n, "calls_of": cap,
                     "distinct_sizes": len(set(shapes)), "batch": f"{bw}x{bh}",
                     "ms_per_candidate": {m: {"median": round(statistics.median(v), 4), "min": round(min(v), 4),
                                              "max": round(max(v), 4)} for m, v in ms.items()},
                     "h2d_kib_per_candidate": {m: round(h2d[m] / 1024, 1) for m in ("set_host", "sizes_host")},
                     "scores_identical": all(v == scores["set_cuda"] for v in scores.values()),
                     "device_memory": memory}
    return out


if __name__ == "__main__":
    main()
