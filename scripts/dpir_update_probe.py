"""DoublePIR entry updates on one GPU: b200pir_dpir_server_update against reloading the whole database.

For 2^30 and 2^33 one-bit entries at pick_params' shapes (n = 1024, p = 512, m = 65536), this times a load of the database
(the second of two, so that module loading is not counted), then for batches of 1, 16, 256, 4096 and 65536 random distinct
entries times update() (wall clock around a call that synchronises; median of --reps after one warm-up call, each call a fresh random batch) and reports entries/s.  A separate
torch.profiler run per batch breaks one update down into device time: store patch, dh_1, digits, hint GEMM (operand images,
A_2 gather, GEMM and add) and the hint's two copies.  Prints one JSON line with the card's name and power limit, and writes it
to --out if given.  Needs a GPU.

    python scripts/dpir_update_probe.py [--sizes 30,33] [--batches 1,16,256,4096,65536] [--reps 5] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

L_FOR = {30: 1821, 33: 14564}       # l = ceil(entries / 9 / 65536)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


STAGES = [("store", ("k_dpir_upd_store",)), ("dh1", ("k_dpir_upd_dh1",)), ("digits", ("k_dpir_upd_digits",)),
          ("hint_gemm", ("k_dpir_upd_gather_a2", "k_gemm_a_image", "k_gemm_b_image", "k_dpir_gemm", "k_dpir_upd_add"))]


def device_split(srv, idx, vals, h2):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        h2 = srv.update(idx, vals, h2)
        torch.cuda.synchronize()
    ev = [(e.name, e.device_time_total / 1e3) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    out = {k: round(sum(t for n, t in ev if any(s in n for s in names)), 3) for k, names in STAGES}
    out["hint_upload"] = round(max([t for n, t in ev if "HtoD" in n] or [0.0]), 3)      # the largest upload is the hint
    out["hint_download"] = round(sum(t for n, t in ev if "DtoH" in n), 3)
    return out, h2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="30,33")
    ap.add_argument("--batches", default="1,16,256,4096,65536")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    import sdk_b200.doublepir as D
    res = dict(card=card(), sizes={})
    for lg in [int(s) for s in a.sizes.split(",")]:
        num_entries = 1 << lg
        prm = dict(n=1024, l=L_FOR[lg], m=65536, logq=32, p=512)
        rng = np.random.default_rng(lg)
        data = rng.integers(0, 256, num_entries // 8, dtype=np.uint8)
        for _ in range(2):                                         # the second load is timed: the first loads the modules
            t0 = time.perf_counter()
            dbm, out, _ = D.load(prm, num_entries, 1, data, D.ENTRY_BITS)
            load_s = time.perf_counter() - t0
        del data
        srv = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, num_entries, 1, max_queries=1)
        h2 = out["h2"]
        row = dict(l=prm["l"], load_s=round(load_s, 3), batches={})
        for k in [int(b) for b in a.batches.split(",")]:
            def batch():
                idx = np.unique(rng.integers(0, num_entries, k + k // 8 + 8, dtype=np.uint64))
                idx = rng.permutation(idx)[:k]
                return idx, rng.integers(0, 2, idx.size, dtype=np.uint8)
            h2 = srv.update(*batch(), h2)                          # warm-up: scratch for this batch size
            times = []
            for _ in range(a.reps):
                idx, vals = batch()
                t0 = time.perf_counter()
                h2 = srv.update(idx, vals, h2)
                times.append(time.perf_counter() - t0)
            med = float(np.median(times))
            split, h2 = device_split(srv, *batch(), h2)
            row["batches"][k] = dict(median_ms=round(med * 1e3, 3), min_ms=round(min(times) * 1e3, 3),
                                     entries_per_s=round(k / med, 1), vs_load=round(med / load_s, 4), device_ms=split)
        res["sizes"][lg] = row
        srv.close()
        dbm.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
