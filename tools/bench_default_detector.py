"""Throughput of the default detector (DBNet-ResNet34) on 2048x1536 synthetic pages at detect_size 2048, one JSON line:

  device_pages_per_s   bilateral pre-filter + network on a device-resident page (CUDA events, after warm-up)
  plugin_pages_per_s   DefaultDetector.infer end to end (host post-processing and copies included)
  kernel_classes       per-class kernel time of one network forward (mitb_profile_report, a separate profiled pass)
  eager_torch          the oracle restatement (oracle/dbnet_r34.py) as eager PyTorch on the same GPU with cuDNN: with the reference's TF32
                       flags (manga_translator.py:135-138) and in plain fp32
  gpu                  card name, power limit and SM clock read in the same run

    python tools/bench_default_detector.py [--pages 8] [--warmup 2]

Weights: the seeded hardened state dict with conv_db.binarize.6.bias lowered (random weights otherwise emit box noise).
"""
import argparse
import asyncio
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "manga-image-translator_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mit_b200 import plugins, synth  # noqa: E402
from mit_b200.engine import get_engine  # noqa: E402
from oracle import dbnet_r34 as r34  # noqa: E402
from oracle import ref_pins_default_detector as pins  # noqa: E402

H, W, DETECT_SIZE = 2048, 1536, 2048


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, power, sm, sm_max = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(sm_max)}
    except Exception as ex:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "error": str(ex)}


def timed(fn, pages, warmup):
    for i in range(warmup):
        fn(pages[i % len(pages)])
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for p in pages:
        fn(p)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("bench_default_detector: needs a CUDA device")
    sd = pins.glue_weights()
    host_pages = [synth.make_page(i, H, W)[0] for i in range(args.pages)]
    eng = get_engine("cuda:0")
    res = {"workload": f"default detector, {args.pages} synthetic {H}x{W} pages, detect_size {DETECT_SIZE}", "gpu": gpu_info()}

    # device resident: bilateral + network (what DefaultDetector._infer runs on the device when the page needs no resize)
    eng.load_dbnet_r34(sd)
    dev_pages = [eng.h2d(p) for p in host_pages]

    def device_step(p):
        return eng.dbnet_r34_forward(eng.bilateral17(p)[None])
    t = timed(device_step, dev_pages, args.warmup)
    res["device_pages_per_s"] = round(args.pages / t, 3)
    res["device_ms_per_page"] = round(1000 * t / args.pages, 3)

    # per-class kernel time of one network forward, in a pass of its own
    x = eng.bilateral17(dev_pages[0])[None]
    eng.profile(True)
    eng.dbnet_r34_forward(x)
    torch.cuda.synchronize()
    rep = eng.profile_report()
    eng.profile(False)
    res["kernel_classes"] = rep

    # the plugin end to end
    plugins.DefaultDetector.set_state_dict(sd)
    det = plugins.DefaultDetector()
    asyncio.run(det.load("cuda:0"))
    for i in range(args.warmup):
        asyncio.run(det.infer(host_pages[i % len(host_pages)], DETECT_SIZE, 0.5, 0.7, 2.3))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n_lines = 0
    for p in host_pages:
        lines, _, _ = asyncio.run(det.infer(p, DETECT_SIZE, 0.5, 0.7, 2.3))
        n_lines += len(lines)
    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    res["plugin_pages_per_s"] = round(args.pages / t, 3)
    res["plugin_lines_per_page"] = round(n_lines / args.pages, 1)
    asyncio.run(det.unload())
    plugins.DefaultDetector.set_state_dict(None)

    # eager PyTorch bar: the oracle's network on the GPU (cuDNN), the caller's /127.5 - 1 and sigmoid included
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    xs = [(p.float() / 127.5 - 1.0).permute(2, 0, 1)[None].contiguous() for p in dev_pages]

    def eager(x):
        db, mask = r34.forward(sd_dev, x)
        return db.sigmoid(), mask
    bar = {}
    for label, tf32 in (("tf32", True), ("fp32", False)):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cudnn.benchmark = False
        t = timed(eager, xs, args.warmup)
        bar[label] = {"pages_per_s": round(args.pages / t, 3), "ms_per_page": round(1000 * t / args.pages, 3)}
    res["eager_torch"] = bar
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
