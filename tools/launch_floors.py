#!/usr/bin/env python3
"""Per-launch-class table of the wgmma engine from PF_PROFILE_CSV dumps, with each class's hardware floor.

    PF_PROFILE_CSV=/tmp/base.csv python bench.py --steps 10      # one dump per build (pf_profile_read writes it)
    python tools/launch_floors.py --steps 10 /tmp/base.csv [/tmp/new.csv ...]

A class is (engine mode, M, N, K, groups).  Its floor per launch is max(MMA time, HBM time):
  MMA time  = 3 bf16 products x 2 M N K groups FLOP / 989 TFLOP/s (H100 SXM data-sheet dense bf16 peak)
  HBM time  = (A hi + lo planes read once, 4 B per element, + weight hi + lo planes, + one 4 B output per element) / 3.35 TB/s
The output term is the least any epilogue writes (one fp32 tensor or one pair of bf16 planes), so the floor is a lower bound.
Times are ms per step; dumps of several builds are shown side by side in the order given."""
import argparse
import csv
from collections import OrderedDict

PEAK_MMA = 989e12
PEAK_HBM = 3.35e12
MODES = {"5": "gemm", "6": "halo"}


def read(path, steps):
    classes = OrderedDict()
    with open(path) as f:
        for r in csv.DictReader(f):
            mode = MODES.get(r["engine_cfg"], r["engine_cfg"])
            M, N, K, groups, cin = int(r["M"]), int(r["N"]), int(r["K"]), int(r["groups"]), int(r["Cin"])
            key = (mode, M, N, K, groups)
            c = classes.setdefault(key, {"launches": 0, "ms": 0.0, "cin": cin})
            c["launches"] += 1
            c["ms"] += float(r["ms"])
    for c in classes.values():
        c["launches"] /= steps
        c["ms"] /= steps
    return classes


def floor_ms(mode, M, N, K, groups, cin):
    flops = 2.0 * M * N * K * groups
    a_elems = M * (cin if mode == "halo" else K) * groups
    nbytes = 4.0 * (a_elems + N * K * groups + M * N * groups)
    mma, hbm = 3 * flops / PEAK_MMA * 1e3, nbytes / PEAK_HBM * 1e3
    return max(mma, hbm), "mma" if mma >= hbm else "hbm", flops, nbytes


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=1, help="steps the dump covers (bench.py --steps)")
    ap.add_argument("--top", type=int, default=0, help="show only the N classes with the most time in the first dump")
    ap.add_argument("csv", nargs="+")
    args = ap.parse_args()
    dumps = [read(p, args.steps) for p in args.csv]
    keys = list(dumps[0])
    for d in dumps[1:]:
        keys += [k for k in d if k not in keys]
    keys.sort(key=lambda k: -dumps[0].get(k, {"ms": 0.0})["ms"])
    if args.top:
        keys = keys[:args.top]
    names = [f"ms[{i}]" for i in range(len(dumps))]
    print(f"{'mode':5} {'M':>8} {'N':>5} {'K':>5} {'g':>2} {'n/step':>6} " + " ".join(f"{n:>9}" for n in names)
          + f" {'floor':>8} {'bound':>5} " + " ".join(f"{'x' + n[2:]:>9}" for n in names))
    tot = [0.0] * len(dumps)
    tot_floor = 0.0
    per_mode = {}
    for k in keys:
        mode, M, N, K, groups = k
        first = next(d[k] for d in dumps if k in d)
        fl, bound, _, _ = floor_ms(mode, M, N, K, groups, first["cin"])
        n = first["launches"]
        ms = [d[k]["ms"] if k in d else float("nan") for d in dumps]
        for i, v in enumerate(ms):
            if v == v:
                tot[i] += v
                per_mode.setdefault(mode, [0.0] * len(dumps))[i] += v
        tot_floor += fl * n
        per_mode.setdefault(mode + " floor", [0.0])[0] += fl * n
        print(f"{mode:5} {M:8d} {N:5d} {K:5d} {groups:2d} {n:6.1f} " + " ".join(f"{v:9.3f}" for v in ms)
              + f" {fl * n:8.3f} {bound:>5} " + " ".join(f"{v / (fl * n):9.2f}" for v in ms))
    print("total ms/step:", " ".join(f"{v:.3f}" for v in tot), f"floor {tot_floor:.3f}")
    for m, v in sorted(per_mode.items()):
        print(f"  {m}:", " ".join(f"{x:.3f}" for x in v))


if __name__ == "__main__":
    main()
