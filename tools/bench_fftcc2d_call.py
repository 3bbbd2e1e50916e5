"""The FFTCC2D call alone on the GPU: bench.py's workload for a 2D config (default B), the queue resident on the device, the
L2 flushed before every call, CUDA events around ocb_fftcc2d_dev.  Prints one line per library:

    <label> fftcc_ms mean M min M max M md5 H

H is the md5 of the records the last call left, so that libraries selected with OCB_LIB_PATH can be compared by their results as
well as their times.  Alternate libraries in separate processes (the library is chosen when the package is imported):

    for i in 1 2 3; do for v in default parent; do
      OCB_LIB_PATH=... python tools/bench_fftcc2d_call.py --label $v; done; done
"""
import argparse
import hashlib
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="B")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--label", default="default")
    args = ap.parse_args()

    import torch
    import opencorr_b200 as ob
    from opencorr_b200 import synth

    if not torch.cuda.is_available():
        sys.exit("no CUDA device: the FFT-CC call is only timed on the GPU")
    cfg = synth.CONFIGS[args.config]
    if cfg["kind"] != "2d":
        sys.exit("config %s is not a 2D workload" % args.config)
    dev = torch.device("cuda", 0)
    ref, tar = synth.speckle_pair_2d(*cfg["size"], second_order=(cfg["order"] == 2), device=dev)
    q0 = ob.make_poi2d(synth.grid_2d(*cfg["grid"]))
    n, r = q0.shape[0], cfg["r"]

    eng = ob.Engine(0)
    stream = torch.cuda.current_stream(dev)
    eng.set_stream(stream.cuda_stream)
    d_ref, d_tar = torch.from_numpy(ref).to(dev), torch.from_numpy(tar).to(dev)
    eng.set_images_2d_dev(d_ref.data_ptr(), d_tar.data_ptr(), ref.shape[1], ref.shape[0])
    d_q0 = torch.from_numpy(q0).to(dev)
    d_q = torch.empty_like(d_q0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)  # 256 MiB > the 50 MB L2

    def call(ev=None):
        d_q.copy_(d_q0)
        flush.zero_()
        if ev:
            ev[0].record(stream)
        eng.fftcc2d_dev(d_q.data_ptr(), n, r, r)
        if ev:
            ev[1].record(stream)

    for _ in range(args.warmup):
        call()
    torch.cuda.synchronize(dev)
    ms = []
    for _ in range(args.calls):
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        call(ev)
        ev[1].synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    md5 = hashlib.md5(d_q.cpu().numpy().tobytes()).hexdigest()
    print("%-8s fftcc_ms mean %.4f min %.4f max %.4f md5 %s" % (args.label, statistics.mean(ms), min(ms), max(ms), md5))


if __name__ == "__main__":
    main()
