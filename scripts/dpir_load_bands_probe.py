"""DoublePIR's banded load on one GPU: `load` against another build of the library, and `load_file` past the old limit.

  --compare DIR   times `load` of 2^24, 2^30 and 2^33 one-bit entries (load_data_fast's input; pick_params' shapes, n = 1024)
                  in this tree and in the tree DIR (another build, e.g. the parent commit's), alternating the two in fresh
                  processes; each process loads once to warm up, then times --reps loads (wall clock; the call synchronises
                  its stream before it returns) and reports a SHA-256 of the last load's outputs (store, h1_squished, a2_t, h2).
  --big           writes a seeded file of 2^36, 2^37 and 2^38 one-bit entries to --dir (removed again), times `load_file` of it
                  (wall clock, ending in a device synchronise) while a second thread samples cudaMemGetInfo every 2 ms (the
                  peak is the largest drop of free device memory below what was free before the call), and at 2^37 gives the
                  device time per stage of one load under torch.profiler.  A size whose file or store does not fit is reported
                  as not measured, with the figures.
Prints one JSON line per measurement and a summary line; --out also writes the summary.

    python scripts/dpir_load_bands_probe.py --compare ../parent [--reps 3] [--big] [--dir /tmp] [--out result.json]
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GIB = 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def params_for(lg):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_oracle_doublepir_e2e as E
    return {k: int(v) for k, v in E.pick_params(1 << lg, 1, E.SEC_PARAM, E.LOGQ).items() if k in ("n", "l", "m", "logq", "p")}


def worker(lg, reps):
    """one tree's load, timed (run with the tree's root first on sys.path)"""
    import sdk_b200.doublepir as D
    prm = json.loads(os.environ["DPIR_PROBE_PRM"])
    data = np.random.default_rng(lg).integers(0, 256, (1 << lg) // 8, dtype=np.uint8)
    dbm, out, _ = D.load(prm, 1 << lg, 1, data, D.ENTRY_BITS)
    dbm.close()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        dbm, out, _ = D.load(prm, 1 << lg, 1, data, D.ENTRY_BITS)
        ms.append(round((time.perf_counter() - t0) * 1e3, 1))
        sq = dbm.download()
        dbm.close()
    h = hashlib.sha256(sq.tobytes())
    for k in ("h1_squished", "a2_t", "h2"):
        h.update(out[k].tobytes())
    print(json.dumps(dict(ms=ms, digest=h.hexdigest())))


def run_worker(tree, lg, reps, prm):
    env = dict(os.environ, DPIR_PROBE_PRM=json.dumps(prm), PYTHONPATH=tree)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", str(lg), "--reps", str(reps)], cwd=tree, env=env,
                       capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("worker in %s: %s" % (tree, r.stderr[-2000:]))
    return json.loads(r.stdout.strip().splitlines()[-1])


def compare(other, reps):
    rows = []
    for lg in (24, 30, 33):
        prm = params_for(lg)
        res = {"this": [], "other": []}
        digests = set()
        for _ in range(3):                                    # alternate: other, this, other, this, ...
            for name, tree in (("other", other), ("this", ROOT)):
                w = run_worker(tree, lg, reps, prm)
                res[name] += w["ms"]
                digests.add(w["digest"])
        row = dict(log2_entries=lg, l=prm["l"], m=prm["m"], p=prm["p"], this_load_ms=res["this"], other_load_ms=res["other"],
                   identical=len(digests) == 1)
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


def write_seeded(path, nbytes, seed):
    chunk = 256 << 20
    with open(path, "wb") as f:
        for k, off in enumerate(range(0, nbytes, chunk)):
            f.write(np.random.default_rng([seed, k]).bytes(min(chunk, nbytes - off)))


STAGES = [("derive", ("k_dpir_derive",)), ("layout", ("k_dpir_layout",)), ("squish", ("k_dpir_add_squish",)),
          ("expand", ("k_dpir_transpose_expand_concat", "k_dpir_pad_transpose"))]


def stage_ms(fn):
    """device time per stage of fn() (one load) from torch.profiler's CUDA records"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    kernels = [(e.name, e.device_time_total / 1e3) for e in ev]
    out = {k: round(sum(t for n, t in kernels if any(s in n for s in names)), 3) for k, names in STAGES}
    gemm = [(n, t) for n, t in kernels if "k_gemm_" in n or "k_dpir_gemm" in n]
    # a_1's image first, then each band's a image and GEMM; the last b image starts h_2's GEMM
    last_b = max(i for i, (n, _) in enumerate(gemm) if "k_gemm_b_image" in n)
    out["gemm_h1"] = round(sum(t for _, t in gemm[:last_b]), 3)
    out["gemm_h2"] = round(sum(t for _, t in gemm[last_b:]), 3)
    out["copies"] = round(sum(t for n, t in kernels if "Memcpy" in n or "Memset" in n), 3)
    out["kernels_total"] = round(sum(t for n, t in kernels if "Memcpy" not in n and "Memset" not in n), 3)
    out["bands"] = sum(1 for n, _ in kernels if "k_dpir_layout" in n)
    return out


def big(dirname):
    import torch
    import sdk_b200.doublepir as D
    rows = []
    for lg in (36, 37, 38):
        prm = params_for(lg)
        l, m, n = prm["l"], prm["m"], prm["n"]
        store = l * ((m + 2) // 3) * 4
        nbytes = (1 << lg) // 8
        torch.cuda.empty_cache()
        free0, total = torch.cuda.mem_get_info()
        row = dict(log2_entries=lg, l=l, m=m, p=prm["p"], store_bytes=store, file_bytes=nbytes)
        disk = shutil.disk_usage(dirname).free
        if disk < nbytes + GIB or free0 < store + 8 * GIB:
            row.update(measured=False, free_disk=disk, free_device=free0)
            print(json.dumps(row), flush=True)
            rows.append(row)
            continue
        path = os.path.join(dirname, "dpir_probe_%d.bin" % lg)
        try:
            t0 = time.perf_counter()
            write_seeded(path, nbytes, lg)
            row["write_s"] = round(time.perf_counter() - t0, 1)
            low = [free0]
            stop = threading.Event()

            def sample():
                while not stop.is_set():
                    low[0] = min(low[0], torch.cuda.mem_get_info()[0])
                    time.sleep(0.002)

            th = threading.Thread(target=sample)
            th.start()
            t0 = time.perf_counter()
            dbm, out, info = D.load_file(prm, 1 << lg, 1, path, D.ENTRY_BITS)
            torch.cuda.synchronize()
            row["load_file_s"] = round(time.perf_counter() - t0, 2)
            stop.set()
            th.join()
            row["peak_device_bytes"] = free0 - low[0]
            row["resident_after_bytes"] = free0 - torch.cuda.mem_get_info()[0]
            dbm.close()
            del out
            if lg == 37:
                torch.cuda.empty_cache()
                row["stages_device_ms"] = stage_ms(lambda: D.load_file(prm, 1 << lg, 1, path, D.ENTRY_BITS)[0].close())
        finally:
            if os.path.exists(path):
                os.remove(path)
        row["measured"] = True
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare", default=None)
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--worker", type=int, default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.worker is not None:
        worker(a.worker, a.reps)
        return
    sys.path.insert(0, ROOT)
    res = dict(card=card())
    if a.compare:
        res["compare"] = compare(os.path.abspath(a.compare), a.reps)
    if a.big:
        res["big"] = big(a.dir)
    line = json.dumps(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
