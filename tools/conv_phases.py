"""Where a tile's time goes in the TMA conv kernel: cycles per tile and consumer warpgroup in four phases (wait on the tile's first
full barrier, main loop, wgmma_wait<0>, epilogue), per GEMM shape, for one device-resident 2048x1536 page.  A staged epilogue is
split further into chunk writes + barriers, column vector loads and the row walk (per-thread clocks averaged over the warpgroup),
and its rows carry the activation, the chain's parts (EpiSig bits) and the signature that ran (512: generic).
MITB_EPI_GENERIC=1 in the environment times the generic signature for an A/B.

Needs the library built with phase timing, which synchronises after every TMA conv launch (so run it on its own, not for times):
  make -C manga-image-translator_b200/csrc clean && make -C manga-image-translator_b200/csrc EXTRA=-DMITB_CONV_PHASES
  python tools/conv_phases.py
and a plain rebuild afterwards."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARK = "conv_phases: timed page"


def child():
    for p in (ROOT, os.path.join(ROOT, "manga-image-translator_b200")):
        sys.path.insert(0, p)
    import torch

    import bench
    from mit_b200 import synth
    from mit_b200.pipeline import HotPath

    torch.set_grad_enabled(False)
    W = bench.build_weights()
    hp = HotPath("cuda:0", W["dbnet"], W["ocr"], W["dictionary"], W["lama"], W["mpe"])
    page, boxes, mask = synth.make_page(0)
    sp = hp.stage(page, synth.make_quads(boxes), mask)
    for _ in range(2):
        hp.run_resident(sp)
    torch.cuda.synchronize()
    sys.stderr.write(MARK + "\n")
    sys.stderr.flush()
    hp.run_resident(sp)
    torch.cuda.synchronize()


def main():
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stderr[-4000:])
        raise SystemExit(f"conv_phases: the page run failed (exit {r.returncode})")
    lines = r.stderr.split(MARK, 1)[-1].splitlines()
    rows = {}
    for ln in lines:
        f = ln.split()
        if not f or f[0] != "mitb_conv_phases":
            continue
        kv = dict(zip(f[1::2], (int(x) for x in f[2::2])))
        key = (kv["M"], kv["K"], kv["N"], kv["BN"], kv["nkb"], kv["act"], kv["parts"], kv["sig"] if kv["staged"] else -1)
        a = rows.setdefault(key, [0] * 9)
        a[0] += 1
        a[1] += kv["tiles"]
        for i, name in enumerate(("first_wait", "main", "wgmma_wait", "epilogue", "epi_chunk", "epi_vec", "epi_rows")):
            a[2 + i] += kv[name]
    if not rows:
        raise SystemExit("conv_phases: no phase records; build the library with EXTRA=-DMITB_CONV_PHASES")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"TMA conv phases, one 2048x1536 page ({gpu}); clk per tile and consumer warpgroup, averaged over the launches of a shape")
    print(f"{'M':>8s} {'K':>6s} {'N':>6s} {'BN':>4s} {'nkb':>4s} {'cnt':>4s} {'wg_tiles':>8s} {'first_wait':>10s} {'main':>8s} {'main/kb':>7s}"
          f" {'wg_wait':>8s} {'epilogue':>8s} {'total':>8s} {'e_chunk':>8s} {'e_vec':>6s} {'e_rows':>8s} {'act':>3s} {'parts':>5s} {'sig':>4s}")
    order = sorted(rows.items(), key=lambda kv: -sum(kv[1][2:6]))
    for (m, k, n, bn, nkb, act, parts, sig), a in order:
        tl = max(1, a[1])
        per = [x / tl for x in a[2:]]
        print(f"{m:8d} {k:6d} {n:6d} {bn:4d} {nkb:4d} {a[0]:4d} {a[1] // a[0]:8d} {per[0]:10.0f} {per[1]:8.0f}"
              f" {per[1] / nkb:7.0f} {per[2]:8.0f} {per[3]:8.0f} {sum(per[:4]):8.0f} {per[4]:8.0f} {per[5]:6.0f} {per[6]:8.0f}"
              f" {act:3d} {parts:5d} {sig:4d}")


if __name__ == "__main__":
    child() if "--child" in sys.argv else main()
