"""DoublePIR offline load on one GPU: b200pir_dpir_load from raw bytes vs b200pir_dpir_setup fed from host memory.

For 2^24, 2^30 and 2^33 one-bit entries (load_data_fast's input: one entry per bit), this times
  * `load`: the raw bytes -> layout, A_1 / A_2 derived on the device -> setup(), database resident in HBM (wall clock);
  * `host setup`: what a host has without it: the l x m layout and both shared matrices in host memory, uploaded through
    b200pir_dpir_setup, which also returns the squished database (wall clock);
alternating the two in one process, checks that their outputs are identical, and breaks one load down into device time per
stage with torch.profiler (kernel durations by name).  Prints one JSON line, and also writes it to --out if given.  Needs a
GPU; the l x m layout for the host path is rebuilt from the squished database the load returns (three 10-bit fields a word).

    python scripts/dpir_load_probe.py [--sizes 24,30,33] [--reps 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# the shapes pick_params gives one-bit entries (n = 1024, p = 512, m = 65536): l = ceil(entries / 9 / 65536)
L_FOR = {24: 29, 30: 1821, 33: 14564}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def unsquish(sq, l, m, p):
    """squish.rs:52-70 inverted for words whose fields are 10 bits: the layout (centred, wrapping u32)."""
    out = np.empty((l, sq.shape[1] * 3), dtype=np.uint32)
    for k in range(3):
        np.right_shift(sq, np.uint32(10 * k), out=out[:, k::3])
        out[:, k::3] &= np.uint32(1023)
    out = np.ascontiguousarray(out[:, :m])
    out -= np.uint32(p // 2)
    return out


STAGES = [("derive", ("k_dpir_derive",)), ("layout", ("k_dpir_layout",)), ("squish", ("k_dpir_add_squish",)),
          ("expand", ("k_dpir_transpose_expand_concat", "k_dpir_pad_transpose"))]


def stage_ms(D, prm, data):
    """Device time per stage of one load, from torch.profiler's CUDA kernel records."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        dbm, _, _ = D.load(prm, len(data) * 8, 1, data, D.ENTRY_BITS)
        torch.cuda.synchronize()
    dbm.close()
    kernels = [(e.name, e.device_time_total / 1e3) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    out = {k: round(sum(t for n, t in kernels if any(s in n for s in names)), 3) for k, names in STAGES}
    gemm = [(n, t) for n, t in kernels if "k_gemm_" in n or "k_dpir_gemm" in n]
    # launch order: a image, b image, GEMM launches of h_1; then the same for h_2
    split = [i for i, (n, _) in enumerate(gemm) if "k_gemm_a_image" in n]
    if len(split) == 2:
        out["gemm_h1"] = round(sum(t for _, t in gemm[:split[1]]), 3)
        out["gemm_h2"] = round(sum(t for _, t in gemm[split[1]:]), 3)
    out["copies"] = round(sum(t for n, t in kernels if "Memcpy" in n or "Memset" in n), 3)
    out["kernels_total"] = round(sum(t for n, t in kernels if "Memcpy" not in n and "Memset" not in n), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="24,30,33")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import sdk_b200.doublepir as D
    res = dict(card=card(), sizes=[])
    for lg in (int(s) for s in a.sizes.split(",")):
        prm = dict(n=1024, l=L_FOR[lg], m=65536, logq=32, p=512)
        data = np.random.default_rng(lg).integers(0, 256, (1 << lg) // 8, dtype=np.uint8)
        dbm, out, info = D.load(prm, 1 << lg, 1, data, D.ENTRY_BITS)            # warm-up, and the host path's inputs
        sq = dbm.download()
        dbm.close()
        db = unsquish(sq, prm["l"], prm["m"], prm["p"])
        a_1 = D.derive_from_seed(prm["m"], prm["n"], D.SEED_A1)
        a_2 = D.derive_from_seed(prm["l"] // info["x"], prm["n"], D.SEED_A2)
        ref = D.setup(db, a_1, a_2, prm["p"], info["delta"], info["x"])         # warm-up
        same = bool(np.array_equal(ref["db_squished"], sq) and all(np.array_equal(ref[k], out[k]) for k in ("h1_squished", "a2_t", "h2")))
        t_load, t_host = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            dbm, out2, _ = D.load(prm, 1 << lg, 1, data, D.ENTRY_BITS)
            t_load.append((time.perf_counter() - t0) * 1e3)
            sq2 = dbm.download()
            dbm.close()
            t0 = time.perf_counter()
            ref2 = D.setup(db, a_1, a_2, prm["p"], info["delta"], info["x"])
            t_host.append((time.perf_counter() - t0) * 1e3)
            same = same and bool(np.array_equal(sq2, ref2["db_squished"]) and all(np.array_equal(out2[k], ref2[k]) for k in ("h1_squished", "a2_t", "h2")))
            del ref2, out2, sq2
        try:
            stages = stage_ms(D, prm, data)
        except Exception as e:                                                    # the timings above stand on their own
            stages = dict(error=str(e))
        res["sizes"].append(dict(log2_entries=lg, l=prm["l"], m=prm["m"], raw_bytes=int(data.size), load_ms=[round(t, 1) for t in t_load],
                                 host_setup_ms=[round(t, 1) for t in t_host], identical=same, load_stage_device_ms=stages))
        del db, a_1, a_2, ref, sq
        print(json.dumps(res["sizes"][-1]), flush=True)
    line = json.dumps(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
