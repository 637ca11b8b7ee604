"""A/B of two builds of libt2h.so on the headline workload (bench.py config 2: vqvae_top encode -> quantize -> decode).

  python tools/ab_headline.py OLD/libt2h.so NEW/libt2h.so [--runs 3] [--steps 20] [--warmup 3] [--batch 16]
                              [--launches] [--out DIR]

The two builds alternate, `--runs` times each, one child process per run: the child points _lib.LIB_PATH at its build
before _lib.load(), builds the step from bench.py's own pieces (VQVAE_TOP, make_inputs, forward_step, ClockSampler,
ops.profile_tapgemm) and prints one JSON line.  Per run: img/s, ms per step, the summed CUDA-event time of the step's
tap-GEMM launches, the median SM clock and the throttle reasons seen during the timed steps.  The card's name, power
limit and maximum SM clock are printed once; a number without them says little.  The last timed step's decoded images
and loss are dumped per build and compared: max |difference|.  `--launches` also runs tools/bench_tapgemm.py once per
build.  Without a CUDA device the script fails; there is no fallback.

The old build is made from the commit to compare against, in a checkout of its own (`git worktree add DIR COMMIT`,
`make -C DIR/text2human_b200/csrc`); no switch selects an older schedule inside one library.
"""
import argparse
import json
import os
import runpy
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(args):
    import contextlib

    import torch

    import bench
    from text2human_b200 import _lib, ops
    _lib.LIB_PATH = os.path.abspath(args.child)
    assert torch.cuda.is_available(), "ab_headline.py needs a CUDA device"
    _lib.load()
    if args.launches:
        runpy.run_path(os.path.join(ROOT, "tools", "bench_tapgemm.py"), run_name="__main__")
        return
    from text2human_b200.pipeline import VQImageSegmTextureModel
    dev = torch.device("cuda", 0)
    ops.set_precision("fp32")
    torch.manual_seed(2021)
    with contextlib.redirect_stdout(sys.stderr):
        model = VQImageSegmTextureModel(bench.VQVAE_TOP).to(dev).eval()
    xs, ms = bench.make_inputs(args.batch, 3, 100)
    xs, ms = [x.to(dev) for x in xs], [m.to(dev) for m in ms]
    for i in range(args.warmup):
        model.forward_step(xs[i % 3], ms[i % 3])
    torch.cuda.synchronize()
    clocks = bench.ClockSampler(0)
    clocks.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        dec, loss = model.forward_step(xs[i % 3], ms[i % 3])
    e1.record()
    torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / args.steps
    clk = clocks.stop()
    ops.profile_tapgemm(True)
    model.forward_step(xs[0], ms[0])
    torch.cuda.synchronize()
    rec = ops.profile_records()
    ops.profile_tapgemm(False)
    bench.dump_outputs(args.dump, dec=dec, loss=loss)
    print(json.dumps(dict(img_per_s=args.batch / (ms_step / 1e3), ms_per_step=ms_step,
                          tapgemm_ms=sum(r[2].elapsed_time(r[3]) for r in rec), tapgemm_launches=len(rec),
                          sm_mhz=clk.get("sm_mhz"), reasons=clk.get("reasons"))), flush=True)


def run_child(so, dump, args, launches=False):
    cmd = [sys.executable, os.path.abspath(__file__), "--child", so, "--dump", dump, "--steps", str(args.steps),
           "--warmup", str(args.warmup), "--batch", str(args.batch)] + (["--launches"] if launches else [])
    out = subprocess.run(cmd, stdout=subprocess.PIPE, text=True, check=True).stdout
    return out if launches else json.loads(out.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("builds", nargs="*", metavar="LIBT2H_SO", help="the old and the new build")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--launches", action="store_true", help="also run tools/bench_tapgemm.py once per build")
    ap.add_argument("--out", default=None, help="directory for the dumped outputs (default: a temporary one)")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    if len(args.builds) != 2:
        ap.error("two libt2h.so paths: the old and the new build")
    for so in args.builds:
        if not os.path.isfile(so):
            ap.error(f"{so}: no such file")
    assert args.runs >= 1 and args.steps >= 1

    import numpy as np
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True, check=True).stdout.strip().splitlines()[0]
    print(f"card: {card} (name, power limit, max SM clock); batch {args.batch}, {args.steps} steps after "
          f"{args.warmup} warm-up steps per run", flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        out = args.out or tmp
        labels = ("old", "new")
        runs = {k: [] for k in labels}
        for r in range(args.runs):
            for label, so in zip(labels, args.builds):
                res = run_child(so, os.path.join(out, label), args)
                runs[label].append(res)
                print(f"run {r} {label}: {res['img_per_s']:7.2f} img/s  {res['ms_per_step']:7.2f} ms/step  tap-GEMM "
                      f"{res['tapgemm_ms']:6.2f} ms in {res['tapgemm_launches']} launches  SM {res['sm_mhz']} MHz  "
                      f"throttle: {','.join(res['reasons']) or 'none'}", flush=True)
        for label in labels:
            v = [x["img_per_s"] for x in runs[label]]
            t = [x["tapgemm_ms"] for x in runs[label]]
            print(f"{label}: img/s {min(v):.2f} .. {max(v):.2f}   tap-GEMM ms {min(t):.2f} .. {max(t):.2f}")
        lo_new, hi_old = min(x["img_per_s"] for x in runs["new"]), max(x["img_per_s"] for x in runs["old"])
        print(f"new's slowest run over old's fastest: {lo_new / hi_old:.4f}")
        for name in ("dec", "loss"):
            a, b = (np.load(os.path.join(out, label, f"{name}.npy")).astype(np.float64) for label in labels)
            print(f"{name}: max |new - old| = {np.abs(a - b).max():.3g} (max |old| = {np.abs(a).max():.3g})")
        if args.launches:
            for label, so in zip(labels, args.builds):
                print(f"--- tools/bench_tapgemm.py, {label} build")
                print(run_child(so, os.path.join(out, label), args, launches=True), end="", flush=True)


if __name__ == "__main__":
    main()
