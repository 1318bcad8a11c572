#!/usr/bin/env python
"""Octave widget levels on the live FIR bank: OctaveSpectrumAnalyzer (one launch per call, levels
only) against the route that existed before it -- Octave_Filters(mode="fft").filter_batch(
want_y=True), one launch per block plus the ragged y gathered with torch.cat, then the widget's
float64 smoothing in torch.  CUDA-event timing after warm-up; prints the card and its power limit.

    python tools/perf_octave_live.py [--channels 1,256,1024] [--bpo 3,24] [--blocks 64]
                                     [--parent-lib OTHER/libfrt_b200.so]

--parent-lib also dumps frt_firbank_process's band outputs y from that build of the library and
from this one on the same seeded input (each in a subprocess, FRT_B200_LIB selects the build),
reports whether they are bit-identical, and times today's route on that build."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP64_PEAK = 34e12      # H100 SXM data sheet, FP64 non-tensor FLOP/s


def dfma_per_channel_block(bpo, block, n_oct=9, L=512):
    """DFMAs the live bank needs per channel and block: bpo band filters on every sample of every
    stage, the decimator on the even samples of every stage but the last."""
    return sum((bpo * (block >> j) + ((block >> j) // 2 if j < n_oct - 1 else 0)) * L for j in range(n_oct))


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the figure is then reported as unknown, not guessed
        pl = "unknown (%s)" % e
    return name, pl


def time_cuda(fn, reps, warmup=2):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3 / reps


def old_route(bank, x, block, alphas_band, decay_band, kernels):
    """Today's route: per-block filter_batch(want_y=True), then float64 smoothing in torch."""
    import torch
    C, T = x.shape
    nb = T // block
    y, _ = bank.filter_batch(x, block=block, energies=False, want_y=True)
    S = torch.stack([(v.view(C, nb, -1).double() ** 2) @ kern for v, kern in zip(y, kernels)], dim=-1)
    sp = torch.zeros((C, len(y)), dtype=torch.float64, device=x.device)
    out = []
    for b in range(nb):
        sp = alphas_band * S[:, b] + sp * decay_band
        out.append(sp)
    return (10 * torch.log10(torch.stack(out, dim=1) + 1e-30)).float()


def old_route_setup(C, bpo, block, n_blocks):
    import torch
    from friture_b200.octavefilters import Octave_Filters, smoothing_alphas
    g = torch.Generator(device="cuda").manual_seed(C * 100 + bpo)
    x = torch.randn((C, n_blocks * block), generator=g, device="cuda") * 0.1
    bank = Octave_Filters(bpo, mode="fft")
    a = smoothing_alphas(1.0)
    decs = bank.get_decs()
    j_of = [int(np.log2(d)) for d in decs]
    alphas_band = torch.tensor([a[j] for j in j_of], dtype=torch.float64, device="cuda")
    decay_band = torch.tensor([(1 - a[j]) ** (block >> j) for j in j_of], dtype=torch.float64, device="cuda")
    kernels = [torch.tensor((1 - a[j]) ** np.arange((block >> j) - 1, -1, -1), dtype=torch.float64,
                            device="cuda") for j in j_of]
    return x, bank, alphas_band, decay_band, kernels


def time_old_route(C, bpo, block, n_blocks, reps):
    x, bank, alphas_band, decay_band, kernels = old_route_setup(C, bpo, block, n_blocks)
    return time_cuda(lambda: old_route(bank, x, block, alphas_band, decay_band, kernels), reps)


def bench(C, bpo, block, n_blocks, reps):
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    x, bank, alphas_band, decay_band, kernels = old_route_setup(C, bpo, block, n_blocks)
    an = OctaveSpectrumAnalyzer(C, bandsperoctave=bpo)     # its own handle, so its own filter plan

    def new():
        an.process(x, block=block)

    def old():
        old_route(bank, x, block, alphas_band, decay_band, kernels)

    an.reset()
    ref_new = an.process(x, block=block).cpu().numpy().astype(np.float64)
    bank.reset()
    ref_old = old_route(bank, x, block, alphas_band, decay_band, kernels).cpu().numpy().astype(np.float64)
    agree = float(np.max(np.abs(ref_new - ref_old)) / max(np.max(np.abs(ref_old)), 1.0))
    t_new = time_cuda(new, reps)
    t_old = time_cuda(old, reps)
    dfma = dfma_per_channel_block(bpo, block)
    share = 2.0 * dfma * C * n_blocks / t_new / FP64_PEAK
    return {"C": C, "bpo": bpo, "block": block, "n_blocks": n_blocks,
            "new_ms": t_new * 1e3, "old_ms": t_old * 1e3, "speedup": t_old / t_new,
            "new_channel_blocks_per_s": C * n_blocks / t_new, "old_channel_blocks_per_s": C * n_blocks / t_old,
            "dfma_per_channel_block": dfma, "fp64_share_of_34TF": share, "db_rel_diff_new_vs_old": agree}


def trim_signatures():
    """An older build of the library lacks the newer calls; the parent-build runs use none of them."""
    import ctypes
    from friture_b200 import _lib
    lib = ctypes.CDLL(_lib.lib_path())
    for name in [n for n in _lib.SIGNATURES if not hasattr(lib, n)]:
        del _lib.SIGNATURES[name]


def dump_y(path):
    """y of frt_firbank_process (through Octave_Filters(mode="fft")) on seeded input."""
    import torch
    from friture_b200.octavefilters import Octave_Filters
    trim_signatures()
    x = torch.from_numpy((np.random.default_rng(7).standard_normal((8, 8 * 1024)) * 0.1).astype(np.float32)).cuda()
    parts = []
    for bpo, block in ((3, 512), (24, 512), (3, 1024), (1, 4096), (12, 256)):
        y, _ = Octave_Filters(bpo, mode="fft").filter_batch(x, block=block, energies=False, want_y=True)
        parts += [v.cpu().numpy().ravel() for v in y]
    np.save(path, np.concatenate(parts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", default="1,256,1024")
    ap.add_argument("--bpo", default="3,24")
    ap.add_argument("--block", type=int, default=512)
    ap.add_argument("--blocks", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--dump-y", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--old-route-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("perf_octave_live: no CUDA device")
    if args.dump_y:
        dump_y(args.dump_y)
        return
    if args.old_route_only:
        trim_signatures()
        for bpo in [int(v) for v in args.bpo.split(",")]:
            for C in [int(v) for v in args.channels.split(",")]:
                print(json.dumps({"C": C, "bpo": bpo, "old_ms_parent_build":
                                  time_old_route(C, bpo, args.block, args.blocks, args.reps) * 1e3}))
        return
    name, pl = card()
    print("card: %s   power.limit, clocks.max.sm: %s" % (name, pl), flush=True)
    if args.parent_lib:
        with tempfile.TemporaryDirectory() as td:
            outs = []
            for lib in (os.path.abspath(args.parent_lib), None):
                env = dict(os.environ)
                env.pop("FRT_B200_LIB", None)
                if lib:
                    env["FRT_B200_LIB"] = lib
                p = os.path.join(td, "y%d.npy" % len(outs))
                subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump-y", p], env=env)
                outs.append(np.load(p))
            same = outs[0].shape == outs[1].shape and np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
            print(json.dumps({"y_bit_identical_parent_vs_new": bool(same), "n_values": int(outs[1].size)}), flush=True)
        env = dict(os.environ, FRT_B200_LIB=os.path.abspath(args.parent_lib))
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--old-route-only",
                               "--channels", args.channels, "--bpo", args.bpo, "--block", str(args.block),
                               "--blocks", str(args.blocks), "--reps", str(args.reps)], env=env)
        sys.stdout.flush()
    for bpo in [int(v) for v in args.bpo.split(",")]:
        for C in [int(v) for v in args.channels.split(",")]:
            print(json.dumps(bench(C, bpo, args.block, args.blocks, args.reps)))


if __name__ == "__main__":
    main()
