"""Per-row timings for SURVEY section 8(f) rows N1/N2/N4 on bench config B (2048^2, 50 000 POIs, 33x33):
device-resident CUDA-event time of each operator through the C ABI's _dev entry points, next to the CPU oracle
(nproc-1 threads) on a bounded sample.  Writes one JSON line per row; `python tools/bench_rows.py > rows.jsonl`.
Not the headline benchmark (that is bench.py)."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import opencorr_b200 as ob
    from opencorr_b200 import synth
    from oracle import oracle
    from oracle.oracle import Oracle2D

    dev = torch.device("cuda", 0)
    cfg = synth.CONFIGS["B"]
    ref, tar = synth.speckle_pair_2d(*cfg["size"])
    xy = synth.grid_2d(*cfg["grid"])
    n, r = len(xy), 16
    eng = ob.Engine(0)
    stream = torch.cuda.current_stream(dev)
    eng.set_stream(stream.cuda_stream)
    d_ref, d_tar = torch.from_numpy(ref).to(dev), torch.from_numpy(tar).to(dev)
    eng.set_images_2d_dev(d_ref.data_ptr(), d_tar.data_ptr(), ref.shape[1], ref.shape[0])
    q0 = ob.make_poi2d(xy)
    d_q0 = torch.from_numpy(q0).to(dev)
    eng.fftcc2d_dev(d_q0.data_ptr(), n, r, r)   # integer guess shared by every row
    torch.cuda.synchronize()
    q_fft = d_q0.cpu().numpy()
    d_q = torch.empty_like(d_q0)
    eng.icgn2d_prepare()
    eng._ck(eng._lib.ocb_nr2d_prepare(eng._ctx))
    lib, ctx = eng._lib, eng._ctx
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)

    # a converged field for the strain row
    eng.icgn2d1_dev(d_q.copy_(d_q0).data_ptr(), n, r, r, 0.001, 10)
    torch.cuda.synchronize()
    d_conv = d_q.clone()
    d_nan = d_conv.clone()
    d_nan[n // 2, 0] = float("nan")  # one POI without a finite position: never binned, never a neighbour

    rows = {
        "ICGN2D1": (lambda p: lib.ocb_icgn2d1_dev(ctx, p, n, r, r, 0.001, 10.0), d_q0),
        "ICGN2D2": (lambda p: lib.ocb_icgn2d2_dev(ctx, p, n, r, r, 0.001, 10.0), d_q0),
        "ICLM2D1": (lambda p: lib.ocb_iclm2d_dev(ctx, 1, p, n, r, r, 0.001, 10.0, 100.0, 0.1, 10.0), d_q0),
        "ICLM2D2": (lambda p: lib.ocb_iclm2d_dev(ctx, 2, p, n, r, r, 0.001, 10.0, 100.0, 0.1, 10.0), d_q0),
        "NR2D1": (lambda p: lib.ocb_nr2d1_dev(ctx, p, n, r, r, 0.001, 10.0), d_q0),
        "Strain2D(r=20,k=5)": (lambda p: lib.ocb_strain2d_dev(ctx, p, n, 20.0, 5, 0.9, 1), d_conv),
        "Strain2D(r=60,k=5)": (lambda p: lib.ocb_strain2d_dev(ctx, p, n, 60.0, 5, 0.9, 1), d_conv),
        "Strain2D(r=20,k=5,one NaN x)": (lambda p: lib.ocb_strain2d_dev(ctx, p, n, 20.0, 5, 0.9, 1), d_nan),
    }
    o = Oracle2D(ref, tar)
    o.prepare()
    threads = o.threads
    sample = 10000
    cpu = {
        "ICGN2D1": lambda q: o.icgn2d1(q, r, r, 0.001, 10),
        "ICGN2D2": lambda q: o.icgn2d2(q, r, r, 0.001, 10),
        "ICLM2D1": lambda q: o.iclm2d(1, q, r, r, 0.001, 10),
        "ICLM2D2": lambda q: o.iclm2d(2, q, r, r, 0.001, 10),
        "NR2D1": lambda q: o.nr2d1(q, r, r, 0.001, 10),
        "Strain2D(r=20,k=5)": lambda q: oracle.strain(q, 20.0, 5, 0.9, 1),
        "Strain2D(r=60,k=5)": lambda q: oracle.strain(q, 60.0, 5, 0.9, 1),
        "Strain2D(r=20,k=5,one NaN x)": lambda q: oracle.strain(q, 20.0, 5, 0.9, 1),
    }
    o.nr2d1(q_fft[:64].copy(), r, r, 0.001, 10)  # builds the NR tables outside the timed region
    for name, (fn, src) in rows.items():
        for _ in range(3):
            d_q.copy_(src)
            assert fn(d_q.data_ptr()) == 0, eng._lib.ocb_last_error(ctx)
        ts = []
        for _ in range(10):
            d_q.copy_(src)
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn(d_q.data_ptr())
            e1.record(stream)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        res = d_q.cpu().numpy()
        ms = float(np.median(ts))
        if name.startswith("Strain"):
            cq = src.cpu().numpy()      # strain needs the whole queue (neighbour search): time it whole
            t0 = time.perf_counter()
            cpu[name](cq)
            cpu_s = time.perf_counter() - t0
            cpu_rate = n / cpu_s
            note = "%d of %d POIs fitted" % (int((res[:, 20] != 0).sum()), n)
            smp = "all %d POIs" % n
        else:
            cq = q_fft[:sample].copy()
            t0 = time.perf_counter()
            cpu[name](cq)
            cpu_s = time.perf_counter() - t0
            cpu_rate = sample / cpu_s
            it = res[res[:, 16] >= 0, 17]
            note = "mean iterations %.2f, converged %.4f" % (float(it.mean()), float((res[:, 16] >= 0).mean()))
            smp = "first %d POIs (tables prepared outside the timed call)" % sample
        print(json.dumps({"row": name, "workload": "config B: 2048x2048, %d POIs, 33x33, FFT-CC guess" % n, "gpu_ms": ms,
                          "gpu_poi_per_s": n / (ms * 1e-3), "cpu_oracle_poi_per_s": cpu_rate, "cpu_threads": threads,
                          "cpu_sample": smp, "speedup": n / (ms * 1e-3) / cpu_rate, "note": note}), flush=True)


    # EpipolarSearch sweep, the parameters of examples/test_3d_reconstruction_epipolar.cpp:137-150 (radius 150, step 4 ->
    # 75 candidates per POI, ICGN2D1 r=20, conv 0.05, stop 5) on the config-B pair with a rectified geometry (y' = y)
    fm = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32)
    ax = np.array([0, 0, 0], np.float32)
    vp = lambda a: a.ctypes.data
    d_q.copy_(torch.from_numpy(q0).to(dev))
    args = (150, 4, 20, 20, 0.05, 5.0)
    for _ in range(2):
        d_q.copy_(torch.from_numpy(q0).to(dev))
        assert lib.ocb_epipolar_search2d_dev(ctx, d_q.data_ptr(), n, vp(fm), vp(ax), vp(ax), *args) == 0
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        d_q.copy_(torch.from_numpy(q0).to(dev))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        lib.ocb_epipolar_search2d_dev(ctx, d_q.data_ptr(), n, vp(fm), vp(ax), vp(ax), *args)
        e1.record(stream)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    res = d_q.cpu().numpy()
    ms = float(np.median(ts))
    smp = 1000
    cq = q0[:smp].copy()
    t0 = time.perf_counter()
    o.epipolar_search(cq, fm, ax, ax, 150, 4, 20, 20, 0.05, 5)
    cpu_rate = smp / (time.perf_counter() - t0)
    agree = float(np.mean(np.all(res[:smp, 14:16] == cq[:, 14:16], axis=1)))
    print(json.dumps({"row": "EpipolarSearch(radius 150, step 4, ICGN2D1 r=20 conv 0.05 stop 5)", "workload": "config B pair, %d POIs x 75 candidates" % n,
                      "gpu_ms": ms, "gpu_poi_per_s": n / (ms * 1e-3), "gpu_candidates_per_s": 75 * n / (ms * 1e-3),
                      "cpu_oracle_poi_per_s": cpu_rate, "cpu_threads": threads, "cpu_sample": "first %d POIs" % smp,
                      "speedup": n / (ms * 1e-3) / cpu_rate,
                      "note": "matched (ZNCC>0.9) %.4f; same winning candidate as the oracle on the sample: %.4f" % (float((res[:, 16] > 0.9).mean()), agree)}),
          flush=True)


if __name__ == "__main__":
    main()
