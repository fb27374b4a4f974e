"""Spiral over row shards driven from one process (b200pir_db_create_sharded): what sharding costs, and what a file load reads.

  one   S8 (nu_2 = 8, 8 GiB in HBM, synthetic seed) unsharded against G = 2 and 4 shards whose contexts are all on device 0:
        throughput of process_query_batch at 16 and 32 queries, single-query latency of process_query, kernel launches per
        call (b200pir_kernel_launches), and whether every layout's responses equal the unsharded bytes.
  load  The bytes read(2) returns to this process (/proc/self/io rchar) while load_file fills a sharded database (T0 shape,
        G = 4), against the file's size: the file is read once, not once per shard.
  multi With two or more GPUs: S8 over devices [0, 1], and the nu_2 = 9 database (16 GiB packed) over [0, 1]; with eight,
        the S256 geometry over all of them at 128 queries.  A leg that needs more GPUs than are visible prints
        "not measured: N GPU visible" and estimates nothing.  The home device's busy time against the others' is not
        measured by this probe.

Latency and throughput: median wall clock of --reps calls that each synchronise, after a warm-up call.  Prints one JSON line
with the card's name and power limit, and writes it to --out if given.  Needs a GPU.

    python scripts/spiral_shard_probe.py [--reps 10] [--parts one,load,multi] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)

SEED = 0xB1755
# the S8 workload of bench.py, and a small shape for the file-load leg
S8 = dict(n=2, nu_1=9, nu_2=8, p=256, q2_bits=22, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
          db_item_size=8192, version=0)
SMALL = dict(n=3, nu_1=5, nu_2=3, p=256, q2_bits=20, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=56, instances=1,
             db_item_size=18432, version=0)
MODULI = (268369921, 249561089)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


def median_s(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def serve(S, kw, pp_arrays, devices, ref, reps, counts=(16, 32)):
    """One layout: contexts on `devices` (one shard each; a single device means unsharded), filled from SEED."""
    ctxs = [S.Params(device=d, **kw) for d in devices]
    H = ctxs[0]
    db = S.Database(H) if len(devices) == 1 else S.Database.sharded(ctxs)
    db.fill_synthetic(SEED)
    gpp = S.PublicParameters(H, pp_arrays["pack"], pp_arrays["left"], pp_arrays["right"], pp_arrays["conv"])
    out = {"devices": devices}
    for count in counts:
        cts = ref["cts"][:count * 2 * 2048]
        got = S.process_query_batch(H, gpp, cts, db)
        if count not in ref["resp"]:
            ref["resp"][count] = got
        out["equal_bytes_%d" % count] = bool(np.array_equal(got, ref["resp"][count]))
        out["qps_%d" % count] = round(count / median_s(lambda: S.process_query_batch(H, gpp, cts, db), reps), 1)
        k0 = S.LIB.b200pir_kernel_launches()
        S.process_query_batch(H, gpp, cts, db)
        out["launches_%d" % count] = int(S.LIB.b200pir_kernel_launches() - k0)
    q = S.Query(ct=ref["cts"][:2 * 2048])
    out["latency_1_ms"] = round(1e3 * median_s(lambda: S.process_query(H, gpp, q, db), reps), 3)
    k0 = S.LIB.b200pir_kernel_launches()
    S.process_query(H, gpp, q, db)
    out["launches_1"] = int(S.LIB.b200pir_kernel_launches() - k0)
    gpp.close()
    db.close()
    for c in ctxs:
        c.close()
    return out


def geometry(S, kw, queries=32):
    """Seeded public parameters (NTT-form words below both moduli) and query ciphertexts (raw words below q0 * q1): every
    layout answers the same inputs, so their response bytes must agree; nothing is decoded."""
    rng = np.random.default_rng(SEED)
    P = S.Params(**kw)
    pp = {k: rng.integers(0, MODULI[1], P.words[k], dtype=np.uint64) for k in ("pack", "left", "right", "conv")}
    cts = rng.integers(0, MODULI[0] * MODULI[1], queries * 2 * 2048, dtype=np.uint64)
    P.close()
    return kw, pp, {"cts": cts, "resp": {}}


def part_one(S, reps):
    kw, pp, ref = geometry(S, S8)
    return [serve(S, kw, pp, [0] * g, ref, reps) for g in (1, 2, 4)]


def rchar():
    with open("/proc/self/io") as f:
        for line in f:
            if line.startswith("rchar:"):
                return int(line.split()[1])
    return -1


def part_load(S):
    ctxs = [S.Params(**SMALL) for _ in range(4)]
    P = ctxs[0]
    rng = np.random.default_rng(SEED)
    words = rng.integers(0, MODULI[0], P.slices * P.dim0 * P.num_per * 2048, dtype=np.uint64) | \
        (rng.integers(0, MODULI[1], P.slices * P.dim0 * P.num_per * 2048, dtype=np.uint64) << np.uint64(32))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "db.bin")
        words.tofile(path)
        db = S.Database.sharded(ctxs)
        r0 = rchar()
        S.check(S.LIB.b200pir_db_load_file(ctxs[0]._h, db._h, path.encode()))
        read = rchar() - r0
        same = bool(np.array_equal(db.to_words(), words))
        db.close()
    out = {"shards": 4, "file_bytes": int(words.nbytes), "download_equals_file": same}
    out["bytes_read"] = int(read) if r0 >= 0 and read > 0 else "not measured: the rchar counter of /proc/self/io did not move"
    return out


def part_multi(S, reps, ngpu):
    out = {}
    if ngpu < 2:
        out["s8_over_0_1"] = out["nu2_9_over_0_1"] = "not measured: %d GPU visible" % ngpu
    else:
        kw, pp, ref = geometry(S, S8)
        out["s8_over_0_1"] = [serve(S, kw, pp, devs, ref, reps) for devs in ([0], [0, 1])]
        kw, pp, ref = geometry(S, dict(S8, nu_2=9))
        out["nu2_9_over_0_1"] = [serve(S, kw, pp, devs, ref, reps) for devs in ([0, 0], [0, 1])]
    if ngpu < 8:
        out["s256_over_8"] = "not measured: %d GPU visible" % ngpu
    else:
        kw, pp, ref = geometry(S, dict(S8, nu_1=10, nu_2=12), queries=128)      # bench.py's S256 workload
        out["s256_over_8"] = serve(S, kw, pp, list(range(8)), ref, reps, counts=(128,))
    out["home_busy_time"] = "not measured"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--parts", default="one,load,multi")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import sdk_b200.spiral as S
    ngpu = int(S.LIB.b200pir_device_count())
    if ngpu < 1:
        raise SystemExit("needs a GPU")
    parts = a.parts.split(",")
    res = {"card": card(), "gpus_visible": ngpu}
    if "one" in parts:
        res["one"] = part_one(S, a.reps)
    if "load" in parts:
        res["load"] = part_load(S)
    if "multi" in parts:
        res["multi"] = part_multi(S, a.reps, ngpu)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
