"""Plaintext read-back of the HBM database on one GPU, parameter set S8 (1 GiB of items, 8.59 GB in HBM), database format
--format (default 2).

Prints the card's name and power limit, then
  - b200pir_db_read_items latency for 1, 16 and 1024 random items (median of --calls calls, wall time);
  - b200pir_db_save_raw_file (1 GiB) against b200pir_db_save_file (8.59 GB) to --dir, alternated, --reps each (wall time,
    fsync included);
  - b200pir_db_load_raw_file of the raw snapshot into a fresh database, which must download identically to the source;
  - the device time of k_read_items over one whole save (torch.profiler's CUDA activity), against the time to read the
    8.59 GB store once at the HBM rate measured here (a device-to-device copy of 2 GiB, counting read + write bytes).

    python scripts/raw_export_probe.py [--format 2] [--reps 3] [--calls 20] [--dir /tmp] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
S8 = dict(n=2, nu_1=9, nu_2=8, p=256, q2_bits=22, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
          db_item_size=8192, version=0)


def timed(fn, G):
    t0 = time.perf_counter()
    fn()
    G.synchronize()
    return time.perf_counter() - t0


def hbm_rate():
    """Bytes per second of a 2 GiB device-to-device copy, read and write counted."""
    import torch
    a = torch.empty(1 << 31, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        b.copy_(a)
    e1.record()
    e1.synchronize()
    rate = 10 * 2 * a.numel() / (e0.elapsed_time(e1) / 1e3)
    del a, b
    torch.cuda.empty_cache()
    return rate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--format", type=int, default=2, choices=(0, 1, 2))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import sdk_b200.spiral as S
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    card = card.strip().splitlines()[0]
    print("card:", card)
    rec = {"card": card, "params": "S8", "format": args.format, "reps": args.reps}
    rec["hbm_copy_GBps"] = hbm_rate() / 1e9
    print("HBM device-to-device copy: %.0f GB/s (read + write)" % rec["hbm_copy_GBps"])
    G = S.Params(**S8)
    db = S.Database(G, fmt=args.format)
    db.fill_synthetic(1)                     # bytes_per_chunk = 2048: every coefficient is returned, so the save is accepted
    n = G.dim0 * G.num_per
    store = G.slices * n * G.poly_len * 8
    rng = np.random.default_rng(1)
    for count in (1, 16, 1024):
        db.read_items(rng.integers(0, n, count, dtype=np.uint64))
        t = [timed(lambda: db.read_items(rng.integers(0, n, count, dtype=np.uint64)), G) for _ in range(args.calls)]
        rec["read_items_%d_ms" % count] = 1e3 * statistics.median(t)
        print("read_items of %4d random items: %.3f ms" % (count, rec["read_items_%d_ms" % count]))

    raw = os.path.join(args.dir, "raw_export_probe_%d.raw" % os.getpid())
    pre = os.path.join(args.dir, "raw_export_probe_%d.bin" % os.getpid())
    try:
        t_raw, t_pre = [], []
        for _ in range(args.reps):
            t_raw.append(timed(lambda: db.save_raw_file(raw), G))
            t_pre.append(timed(lambda: db.save_file(pre), G))
            os.unlink(pre)                   # one 8.59 GB snapshot on disk at a time
        rec["save_raw_file_s"], rec["save_file_s"] = statistics.median(t_raw), statistics.median(t_pre)
        rec["save_raw_file_all_s"], rec["save_file_all_s"] = t_raw, t_pre
        print("save_raw_file: %.3f s (%.2f GB/s of file)  save_file: %.3f s (%.2f GB/s of file)" %
              (rec["save_raw_file_s"], n * G.db_item_size / rec["save_raw_file_s"] / 1e9, rec["save_file_s"],
               store / rec["save_file_s"] / 1e9))
        assert os.path.getsize(raw) == n * G.db_item_size

        fresh = S.Database(G, fmt=args.format)
        t = [timed(lambda: S.check(S.LIB.b200pir_db_load_raw_file(G._h, fresh._h, raw.encode())), G) for _ in range(args.reps)]
        rec["load_raw_file_s"] = statistics.median(t)
        print("load_raw_file of the raw snapshot: %.3f s" % rec["load_raw_file_s"])
        rec["reload_identical"] = bool(np.array_equal(fresh.to_words(), db.to_words()))
        print("reloaded database downloads identically:", rec["reload_identical"])
        fresh.close()

        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            db.save_raw_file(raw)
            G.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "k_read_items" in e.key)
        rec["k_read_items_s"] = us / 1e6
        rec["store_read_at_hbm_rate_s"] = store / (rec["hbm_copy_GBps"] * 1e9)
        print("k_read_items over one save: %.3f s device time; reading the %.2f GB store at the measured rate: %.4f s" %
              (rec["k_read_items_s"], store / 1e9, rec["store_read_at_hbm_rate_s"]))
    finally:
        for p in (raw, pre):
            if os.path.exists(p):
                os.unlink(p)
    db.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raw_export_probe_f%d.json" % args.format), "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
