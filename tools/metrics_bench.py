"""Time the scoring kernels (csrc/metrics.cuh) with CUDA events against a device-to-device copy, in one process:

    python tools/metrics_bench.py [--iters 20] [--out results/metrics_bench.json]

* ``losses`` of a PersNet-360Cities batch of 32 at 320 x 320 (cross-entropy over 73 + 180 logit planes: 3.3 GB read);
* ``losses`` of a regression variant's batch of 32 at 320 x 320 (multi-scale gradient and L2 terms);
* ``field_errors`` on 256 images of 640 x 480 (statistics only, and with the error maps returned).

Bytes are what each call must read and write, computed from the shapes; a copy that moves as many bytes (reads half, writes half)
is the ceiling.
Prints one JSON object with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_ms(fn, match, reps=3):
    """Per-kernel device time per call of fn, from torch.profiler in a pass of its own (kernels whose name contains match)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return {e.key[:40]: e.device_time_total / 1e3 / reps for e in prof.key_averages() if match in e.key}


def copy_ms(nbytes, iters):
    """A device-to-device copy that reads nbytes (and writes as many)."""
    src = torch.empty(nbytes // 4, dtype=torch.float32, device="cuda")
    dst = torch.empty_like(src)
    return timed(lambda: dst.copy_(src), iters)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit unavailable: {e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench needs a CUDA device")
    import pf_test_util as U
    from perspectivefields_b200 import metrics

    res = {"gpu": gpu_info(), "cases": {}}
    n, h, w = 32, 320, 320
    # classification losses
    m = U.make_model("PersNet-360Cities", seed=0, device="cuda")[0]
    pg = torch.randn((n, 73, h, w), device="cuda")
    pl = torch.randn((n, 180, h, w), device="cuda")
    results = [{"pred_gravity": a, "pred_latitude": b} for a, b in zip(pg.unbind(0), pl.unbind(0))]
    tg = {"gt_gravity": torch.randint(0, 73, (n, h, w), device="cuda"), "gt_latitude": torch.randint(0, 180, (n, h, w), device="cuda")}
    ms = timed(lambda: m.losses(results, tg), args.iters)
    read = (73 + 180) * n * h * w * 4 + 2 * n * h * w * 8
    cms = copy_ms(read // 2, args.iters)                  # a copy of half the bytes moves as many in total
    res["cases"]["losses_classification_b32_320"] = {"ms": ms, "bytes_read": read, "GB_per_s": read / ms / 1e6, "copy_ms_same_traffic": cms,
                                                     "fraction_of_copy_rate": cms / ms,
                                                     "kernel_ms_per_call": kernel_ms(lambda: m.losses(results, tg), "pf::")}
    del pg, pl, results, tg
    # regression losses
    m = U.make_model("Paramnet-360Cities-edina-centered", seed=0, device="cuda")[0]
    v = torch.randn((n, 2, h, w), device="cuda")
    v = v / v.norm(dim=1, keepdim=True)
    results = [{"pred_gravity": a, "pred_latitude": b} for a, b in zip(v.unbind(0), torch.rand((n, 1, h, w), device="cuda").unbind(0))]
    tg = {"gt_gravity": v.flip(1).contiguous(), "gt_latitude": torch.rand((n, 1, h, w), device="cuda")}
    ms = timed(lambda: m.losses(results, tg), args.iters)
    read = 6 * n * h * w * 4
    cms = copy_ms(read // 2, args.iters)                  # a copy of half the bytes moves as many in total
    res["cases"]["losses_regression_b32_320"] = {"ms": ms, "bytes_read": read, "GB_per_s": read / ms / 1e6, "copy_ms_same_traffic": cms,
                                                 "fraction_of_copy_rate": cms / ms,
                                                 "kernel_ms_per_call": kernel_ms(lambda: m.losses(results, tg), "pf::")}
    del v, results, tg
    # field errors
    n, h, w = 256, 480, 640
    pu = torch.randn((n, 2, h, w), device="cuda")
    plat = torch.rand((n, h, w), device="cuda") * 180 - 90
    results = [{"pred_gravity_original": a, "pred_latitude_original": b} for a, b in zip(pu.unbind(0), plat.unbind(0))]
    gu = torch.randn((n, h, w, 2), device="cuda")
    glat = torch.rand((n, h, w), device="cuda") * 180 - 90
    ups, lats = list(gu.unbind(0)), list(glat.unbind(0))
    for maps in (False, True):
        ms = timed(lambda: metrics.field_errors(results, ups, lats, return_maps=maps), max(args.iters // 2, 3))
        moved = 6 * n * h * w * 4 + 2 * n * h * w * 4        # read 6 floats per pixel, write 2 error values (maps or workspace)
        cms = copy_ms(moved // 2, args.iters)                 # a copy of half the bytes moves as many in total
        res["cases"][f"field_errors_256x640x480{'_maps' if maps else ''}"] = {
            "ms": ms, "bytes_moved_error_pass": moved, "GB_per_s_error_pass_equiv": moved / ms / 1e6, "copy_ms_same_traffic": cms,
            "fraction_of_copy_rate": cms / ms, "images_per_s": n / ms * 1e3}
    res["field_errors_kernel_ms_per_call"] = kernel_ms(lambda: metrics.field_errors(results, ups, lats), "pf::")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
