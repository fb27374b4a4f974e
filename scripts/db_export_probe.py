"""Read-back and load rates of the HBM database on one GPU, parameter set S8 (8 GiB in HBM) in database format --format.

Prints the card's name and power limit, then
  - b200pir_db_fill_synthetic and Database.from_words (b200pir_db_upload from a host array), wall time ending in a device
    synchronise (median of --reps runs);
  - b200pir_db_download of the whole database and b200pir_db_save_file to --dir, wall time ending in a device synchronise,
    with GB/s (median of --reps runs);
  - the device time of the un-tiling kernels alone (torch.profiler's CUDA activity of k_db_export_*, summed over one
    download) against their algorithmic traffic (8.59 GB read + 8.59 GB written);
  - b200pir_db_load_file of the saved file;
  - single-query latency (random public parameters and query: no client keys needed) while a save runs, against idle.

    python scripts/db_export_probe.py [--format 2] [--reps 3] [--dir /tmp] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
S8 = dict(n=2, nu_1=9, nu_2=8, p=256, q2_bits=22, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
          db_item_size=8192, version=0)
Q0, Q1 = 268369921, 249561089


def timed(fn, G):
    t0 = time.perf_counter()
    fn()
    G.synchronize()
    return time.perf_counter() - t0


def rand_ntt(rng, words):
    return rng.integers(0, Q0, words, dtype=np.uint64) | (rng.integers(0, Q1, words, dtype=np.uint64) << np.uint64(32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--format", type=int, default=2, choices=(0, 1, 2))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import sdk_b200.spiral as S
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    print("card:", card.strip().splitlines()[0])
    rec = {"card": card.strip().splitlines()[0], "params": "S8", "format": args.format, "reps": args.reps}
    G = S.Params(**S8)
    db = S.Database(G, fmt=args.format)
    db.fill_synthetic(1)                                                   # first fill: the kernel's module is loaded here
    nbytes = G.slices * G.dim0 * G.num_per * G.poly_len * 8
    t = [timed(lambda: db.fill_synthetic(1), G) for _ in range(args.reps)]
    rec["fill_synthetic_s"] = statistics.median(t)
    print("fill_synthetic: %.3f s  %.2f GB/s" % (rec["fill_synthetic_s"], nbytes / rec["fill_synthetic_s"] / 1e9))
    words = np.empty(nbytes // 8, dtype=np.uint64)
    words.fill(0)                                                          # fault the pages in outside the timed window
    db.to_words(out=words)                                                 # first export: staging allocated here
    t = [timed(lambda: db.to_words(out=words), G) for _ in range(args.reps)]
    rec["download_s"] = statistics.median(t)
    rec["download_GBps"] = nbytes / rec["download_s"] / 1e9
    print("download: %.3f s  %.2f GB/s" % (rec["download_s"], rec["download_GBps"]))

    def upload():
        S.Database.from_words(G, words, fmt=args.format).close()

    upload()
    t = [timed(upload, G) for _ in range(args.reps)]
    rec["from_words_s"] = statistics.median(t)
    print("from_words: %.3f s  %.2f GB/s" % (rec["from_words_s"], nbytes / rec["from_words_s"] / 1e9))

    path = os.path.join(args.dir, "db_export_probe_%d.bin" % os.getpid())
    try:
        t = [timed(lambda: db.save_file(path), G) for _ in range(args.reps)]
        rec["save_file_s"] = statistics.median(t)
        rec["save_file_GBps"] = nbytes / rec["save_file_s"] / 1e9
        print("save_file: %.3f s  %.2f GB/s" % (rec["save_file_s"], rec["save_file_GBps"]))
        assert np.array_equal(np.fromfile(path, dtype=np.uint64, count=1 << 20), words[:1 << 20])

        try:
            import torch
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                db.to_words(out=words)
                G.synchronize()
            us = sum(e.device_time_total for e in prof.key_averages() if "k_db_export" in e.key)
            rec["untile_kernel_s"] = us / 1e6
            rec["untile_kernel_GBps"] = 2 * nbytes / (us / 1e6) / 1e9 if us else None
            print("un-tiling kernels: %.3f s over one download, %.0f GB/s of read + write" %
                  (rec["untile_kernel_s"], rec["untile_kernel_GBps"] or 0))
        except Exception as e:                                             # the probe still reports the rest
            print("kernel timing unavailable:", e)

        fresh = S.Database(G, fmt=args.format)
        t = [timed(lambda: S.LIB.b200pir_db_load_file(G._h, fresh._h, path.encode()), G) for _ in range(args.reps)]
        rec["load_file_s"] = statistics.median(t)
        print("load_file: %.3f s  %.2f GB/s" % (rec["load_file_s"], nbytes / rec["load_file_s"] / 1e9))
        fresh.close()

        rng = np.random.default_rng(5)
        pp = S.PublicParameters(G, rand_ntt(rng, G.words["pack"]), rand_ntt(rng, G.words["left"]),
                                rand_ntt(rng, G.words["right"]), rand_ntt(rng, G.words["conv"]))
        qry = S.Query(ct=(rng.integers(0, 2**56, 2 * G.poly_len, dtype=np.uint64)))
        for _ in range(5):
            S.process_query(G, pp, qry, db)

        def latencies(n):
            out = []
            for _ in range(n):
                t0 = time.perf_counter()
                S.process_query(G, pp, qry, db)
                out.append(time.perf_counter() - t0)
            return out

        idle = latencies(50)
        busy, stop = [], threading.Event()

        def saver():
            try:
                db.save_file(path)
            finally:
                stop.set()

        th = threading.Thread(target=saver)
        th.start()
        while not stop.is_set():
            busy += latencies(1)
        th.join()
        rec["query_idle_ms"] = 1e3 * statistics.median(idle)
        rec["query_during_save_ms"] = 1e3 * statistics.median(busy)
        rec["query_during_save_p99_ms"] = 1e3 * sorted(busy)[int(0.99 * (len(busy) - 1))]
        rec["queries_during_save"] = len(busy)
        print("single query: idle %.2f ms, during a save %.2f ms (p99 %.2f ms, %d queries served)" %
              (rec["query_idle_ms"], rec["query_during_save_ms"], rec["query_during_save_p99_ms"], len(busy)))
        pp.close()
    finally:
        if os.path.exists(path):
            os.unlink(path)
    db.close()
    G.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "db_export_probe.json"), "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
