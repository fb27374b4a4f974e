"""Write rate of the database writers on one GPU, parameter set S8 (2^17 items of 8192 bytes, 8 GiB in HBM).

For bodies of 1, 16, 1024 and 2^14 full items to distinct random db_idx it times
  (a) one b200pir_db_update_item_raw call per item, and
  (b) one b200pir_db_update_many_items call on the /update-row body of the same items,
each with a host clock that ends in a device synchronise (median of --reps runs), and prints items/s and body MB/s.  It also
times a full b200pir_db_load_raw_file of a 1 GiB raw S8 file; with --compare ROOT it times the same load with the built
package of another checkout (ROOT/sdk_b200), alternating the two.  Afterwards it checks that the databases written by (a)
and (b) give identical response bytes for queries on written items (random public parameters and queries: the comparison
needs no client keys).  The card's name and power limit are printed first.

    python scripts/update_rate_probe.py [--reps 3] [--compare ROOT] [--out DIR]
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
S8 = dict(n=2, nu_1=9, nu_2=8, p=256, q2_bits=22, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
          db_item_size=8192, version=0)
Q0, Q1 = 268369921, 249561089

# run in a fresh interpreter with sys.path[0] = the package root to time: prints the seconds of one load_raw_file
LOAD_SNIPPET = r"""
import sys, time
sys.path.insert(0, sys.argv[1])
import numpy as np
import sdk_b200.spiral as S
from sdk_b200._lib import LIB, check
G = S.Params(**eval(sys.argv[3]))
db = S.Database(G)
db.update_item_raw(0, np.zeros(1, dtype=np.uint8))   # module load and first launches outside the timed window
G.synchronize()
t0 = time.perf_counter()
check(LIB.b200pir_db_load_raw_file(G._h, db._h, sys.argv[2].encode()))
G.synchronize()
print(time.perf_counter() - t0)
"""


def entry(db_idx, data):
    return (4 + len(data)).to_bytes(4, "big") + int(db_idx).to_bytes(4, "big") + data


def timed(fn, G):
    t0 = time.perf_counter()
    fn()
    G.synchronize()
    return time.perf_counter() - t0


def load_seconds(pkg_root, path):
    out = subprocess.check_output([sys.executable, "-c", LOAD_SNIPPET, pkg_root, path, repr(S8)], text=True)
    return float(out.split()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--compare", help="root of another checkout whose built sdk_b200 times load_raw_file too")
    ap.add_argument("--out", help="directory for the JSON record")
    args = ap.parse_args()
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    print("card:", card.strip().splitlines()[0])
    rec = {"card": card.strip().splitlines()[0], "params": "S8", "reps": args.reps}

    # full load_raw_file of S8, this build (and the compared one), alternating
    rng = np.random.default_rng(2024)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s8.raw")
        num_items = (1 << (S8["nu_1"] + S8["nu_2"]))
        rng.integers(0, 256, num_items * S8["db_item_size"], dtype=np.uint8).tofile(path)
        loads = {"this": []}
        if args.compare:
            loads["compare"] = []
        for _ in range(2):
            loads["this"].append(load_seconds(ROOT, path))
            if args.compare:
                loads["compare"].append(load_seconds(os.path.abspath(args.compare), path))
        for k, v in loads.items():
            print("load_raw_file S8 (%s build): %s s" % (k, " ".join("%.3f" % x for x in v)))
        rec["load_raw_file_s"] = loads

    sys.path.insert(0, ROOT)
    import sdk_b200.spiral as S
    G = S.Params(**S8)
    a, b = S.Database(G), S.Database(G)
    size = S8["db_item_size"]
    a.update_item_raw(0, np.zeros(size, dtype=np.uint8))     # warm both paths
    b.update_many_items(entry(0, bytes(size)))
    rows = []
    for count in (1, 16, 1024, 1 << 14):
        idxs = rng.choice(num_items, count, replace=False)
        items = rng.integers(0, 256, (count, size), dtype=np.uint8)
        datas = [items[k] for k in range(count)]
        body = b"".join(entry(int(i), d.tobytes()) for i, d in zip(idxs, datas))
        ta, tb = [], []
        for _ in range(args.reps):
            ta.append(timed(lambda: [a.update_item_raw(int(i), d) for i, d in zip(idxs, datas)], G))
            tb.append(timed(lambda: b.update_many_items(body), G))
        ma, mb = statistics.median(ta), statistics.median(tb)
        row = dict(items=count, body_bytes=len(body), loop_s=ma, batch_s=mb, loop_items_per_s=count / ma, batch_items_per_s=count / mb,
                   loop_MB_per_s=len(body) / ma / 1e6, batch_MB_per_s=len(body) / mb / 1e6, speedup=ma / mb)
        rows.append(row)
        print("%6d items  (a) loop %10.0f items/s %8.1f MB/s   (b) batch %10.0f items/s %8.1f MB/s   (a)/(b) time %.2fx"
              % (count, row["loop_items_per_s"], row["loop_MB_per_s"], row["batch_items_per_s"], row["batch_MB_per_s"], row["speedup"]))
    rec["writes"] = rows

    # (a) and (b) saw the same items in the same order: the two databases must answer identically
    W = 2 * 2048
    def ntt_mat(polys):
        m = np.empty((polys, 2, 2048), dtype=np.uint64)
        m[:, 0] = rng.integers(0, Q0, (polys, 2048), dtype=np.uint64)
        m[:, 1] = rng.integers(0, Q1, (polys, 2048), dtype=np.uint64)
        return m.reshape(-1)
    pp = S.PublicParameters(G, ntt_mat(G.words["pack"] // W), ntt_mat(G.words["left"] // W), ntt_mat(G.words["right"] // W),
                            ntt_mat(G.words["conv"] // W))
    same = True
    for k in range(4):
        ct = rng.integers(0, Q0 * Q1, 2 * 2048, dtype=np.uint64)
        ra = S.process_query(G, pp, S.Query(ct=ct), a)
        rb = S.process_query(G, pp, S.Query(ct=ct), b)
        same &= bool(np.array_equal(ra, rb))
    print("responses of (a) and (b) identical:", same)
    rec["responses_identical"] = same
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "update_rate_probe.json"), "w") as f:
            json.dump(rec, f, indent=1)
    for h in (pp, a, b, G):
        h.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
