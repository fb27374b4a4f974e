"""DoublePIR answer() on one GPU: the resident server (sdk_b200.doublepir.Server) against the host-buffer chain
(sdk_b200.doublepir.answer), answer_many throughput, and the database pass's kernel time.

For 2^30 and 2^33 one-bit entries (l = 1821 / 14564 rows of 21846 packed words, loaded from seeded bytes with `load`) this
measures, in one process:
  * single-request latency (wall clock, median of --reps, the two paths alternated, outputs asserted identical);
  * answer_many requests/s at 1, 2, 4, 8, 16 and 32 single-query requests (median of --reps calls);
then, in a separate torch.profiler run, kernel times by name:
  * the database pass of one call with V = 1 and V = 16 requests (the first k_dpir_matvec_multi launch of the call), as GB/s
    of the squished database against 3.35 TB/s;
  * matrix_mul_vec_packed_many over the database at V = 1, 2, 4, 8, 16 (where the integer pipe starts to bound the pass);
  * k_dpir_matvec_multi at V = 1 against k_dpir_matvec_wide (the existing dispatch) at l = 29 and at the 2^33 database.
Queries are random vectors of the right lengths: the server's work does not depend on their values.  Prints one JSON line
and also writes it to --out if given.  Needs a GPU.

    python scripts/dpir_answer_probe.py [--sizes 30,33] [--reps 30] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

L_FOR = {24: 29, 30: 1821, 33: 14564}        # pick_params for one-bit entries: n = 1024, p = 512, m = 65536
HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def kernel_times(fn):
    """[(kernel name, device ms)] of everything fn() launches, in launch order"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, e.device_time_total / 1e3) for e in ev]


def median_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="30,33")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import sdk_b200.doublepir as D
    res = dict(card=card(), sizes=[])
    for lg in (int(s) for s in a.sizes.split(",")):
        prm = dict(n=1024, l=L_FOR[lg], m=65536, logq=32, p=512)
        rng = np.random.default_rng(lg)
        data = rng.integers(0, 256, (1 << lg) // 8, dtype=np.uint8)
        dbm, out, info = D.load(prm, 1 << lg, 1, data, D.ENTRY_BITS)
        del data
        n, l, delta, x, ne = prm["n"], prm["l"], info["delta"], info["x"], info["ne"]
        c1 = out["h1_squished"].shape[1]
        qs = [[rng.integers(0, 2**32, 3 * dbm.cols, dtype=np.uint64).astype(np.uint32),
               rng.integers(0, 2**32, 3 * c1, dtype=np.uint64).astype(np.uint32)] for _ in range(32)]
        h_1 = (out["h1_squished"].reshape(-1), n * delta * x, c1)
        a2t = (out["a2_t"].reshape(-1), n, out["a2_t"].shape[1])
        srv = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, 1 << lg, 1, max_queries=32)
        reqs = [D.serialize_request([q]) for q in qs]

        def chain(q):
            msg = D.answer(dbm, [q], h_1, a2t, prm["p"], delta, x, ne)
            return D.serialize_state([msg[0].reshape(delta * x, n)] + msg[1:])

        identical = all(chain(q) == srv.answer(r) for q, r in zip(qs[:4], reqs[:4]))     # also the warm-up
        t_chain, t_srv = [], []
        for k in range(a.reps):
            t_chain.append(median_ms(lambda: chain(qs[k % 32]), 1))
            t_srv.append(median_ms(lambda: srv.answer(reqs[k % 32]), 1))
        many = {}
        for cnt in (1, 2, 4, 8, 16, 32):
            got = srv.answer_many(reqs[:cnt])
            identical = identical and all(g == srv.answer(r) for g, r in zip(got[:2], reqs[:2]))
            ms = median_ms(lambda: srv.answer_many(reqs[:cnt]), max(5, a.reps // 3))
            many[cnt] = dict(call_ms=round(ms, 3), requests_per_s=round(cnt / ms * 1e3, 1))
        db_bytes = l * dbm.cols * 4
        prof = {}
        try:
            for cnt in (1, 16):
                ks = [t for nm, t in kernel_times(lambda: srv.answer_many(reqs[:cnt])) if "k_dpir_matvec_multi" in nm]
                prof["db_pass_V%d" % cnt] = dict(ms=round(ks[0], 4), GBps=round(db_bytes / ks[0] / 1e6, 1),
                                                 hbm_share=round(db_bytes / ks[0] / 1e6 / (HBM_TBS * 1e3), 3))
            for v in (1, 2, 4, 8, 16):
                b = rng.integers(0, 2**32, (v, 3 * dbm.cols), dtype=np.uint64).astype(np.uint32)
                D.matrix_mul_vec_packed_many(dbm, b)
                ks = [t for nm, t in kernel_times(lambda: D.matrix_mul_vec_packed_many(dbm, b)) if "k_dpir_matvec_multi" in nm]
                prof["many_V%d" % v] = dict(ms=round(ks[0], 4), GBps=round(db_bytes / ks[0] / 1e6, 1),
                                            words_per_ns=round(l * dbm.cols / ks[0] / 1e6, 2))
            b1 = qs[0][0]
            for tag, m in (("l29", D.PackedMatrix(rows=29, cols=dbm.cols, synthetic_seed=7)), ("l%d" % l, dbm)):
                D.matrix_mul_vec_packed(m, b1)
                D.matrix_mul_vec_packed_many(m, b1[None])
                assert np.array_equal(D.matrix_mul_vec_packed(m, b1), D.matrix_mul_vec_packed_many(m, b1[None])[0])
                wide = [t for nm, t in kernel_times(lambda: D.matrix_mul_vec_packed(m, b1)) if "k_dpir_matvec_wide" in nm]
                multi = [t for nm, t in kernel_times(lambda: D.matrix_mul_vec_packed_many(m, b1[None])) if "k_dpir_matvec_multi" in nm]
                prof["V1_vs_wide_" + tag] = dict(wide_ms=round(wide[0], 4), multi_ms=round(multi[0], 4))
                if m is not dbm:
                    m.close()
        except Exception as e:                                                    # the timings above stand on their own
            prof["error"] = repr(e)
        srv.close()
        dbm.close()
        res["sizes"].append(dict(log2_entries=lg, l=l, packed_cols=int(dbm.cols), db_mb=round(db_bytes / 1e6, 1), identical=bool(identical),
                                 single_ms=dict(chain=round(float(np.median(t_chain)), 3), server=round(float(np.median(t_srv)), 3)),
                                 answer_many=many, kernels=prof))
        print(json.dumps(res["sizes"][-1]), flush=True)
    line = json.dumps(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
