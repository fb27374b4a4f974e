"""DoublePIR's database pass on the tensor cores (k_dpir_matvec_tc) against the integer kernel (k_dpir_matvec_multi), and
answer_many throughput with the kernel selection in place.

For 2^30 and 2^33 one-bit entries (l = 1821 / 14564 rows of 21846 packed words, loaded from seeded bytes with `load`) this
measures, in one process, with the card's name and power limit:
  * matrix_mul_vec_packed_many over the database at V = 1, 2, 4, 8, 16, 32, 64, 128 on each kernel, alternating the two at each
    V (outputs asserted identical): kernel time from torch.profiler (the pass kernel, and the query-image builder separately),
    as ns per vector-word (a vector-word = one packed word of the matrix against one vector) and as a share of the larger of
    the HBM bound (the squished database once per launch at 3.35 TB/s) and the dense-INT8 bound (8 limb products per digit at
    1979 TOPS, data sheet);
  * answer_many requests/s at 1 .. 128 single-query requests (median wall time of --reps calls), every response asserted equal
    to the request answered alone (which runs the integer kernel);
  * in a separate torch.profiler run, the kernels of one 64-request call by name (count and device time).
Prints one JSON line per size and a final one, also written to --out if given.  Needs a GPU.

    python scripts/dpir_tc_probe.py [--sizes 30,33] [--reps 20] [--out result.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

L_FOR = {24: 29, 30: 1821, 33: 14564}        # pick_params for one-bit entries: n = 1024, p = 512, m = 65536
HBM_TBS = 3.35
INT8_TOPS = 1979.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--vs", default="1,2,4,8,16,32,64,128")
    ap.add_argument("--counts", default="1,2,4,8,16,32,64,128")
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
        l, cols = prm["l"], int(dbm.cols)
        db_bytes = l * cols * 4
        # ---- the pass, both kernels alternating
        passes = {}
        for v in (int(x) for x in a.vs.split(",")):
            b = rng.integers(0, 2**32, (v, 3 * cols), dtype=np.uint64).astype(np.uint32)
            outs = {}
            for kern in (D.MV_MULTI, D.MV_TC):
                outs[kern] = D._matvec_packed_many_on(dbm, b, kern)                      # warm-up
            assert np.array_equal(outs[D.MV_MULTI], outs[D.MV_TC]), v
            row = {}
            for rep in range(2):
                for kern, tag in ((D.MV_MULTI, "multi"), (D.MV_TC, "tc")):
                    ks = kernel_times(lambda: D._matvec_packed_many_on(dbm, b, kern))
                    t = sum(ms for nm, ms in ks if "k_dpir_matvec_multi" in nm or "k_dpir_matvec_tc" in nm)
                    img = sum(ms for nm, ms in ks if "k_dpir_tc_image" in nm)
                    row.setdefault(tag, []).append((t, img))
            entry = {}
            for tag, ts in row.items():
                t = min(x for x, _ in ts)
                img = min(y for _, y in ts)
                hbm_ms = db_bytes / (HBM_TBS * 1e12) * 1e3 * (1 if tag == "tc" else -(-v // 16))
                tc_ms = 2.0 * 8 * l * 3 * cols * v / (INT8_TOPS * 1e12) * 1e3
                bound = max(hbm_ms, tc_ms)
                entry[tag] = dict(kernel_ms=round(t, 4), image_ms=round(img, 4), ns_per_vector_word=round(t * 1e6 / (v * l * cols), 5),
                                  bound="hbm" if hbm_ms >= tc_ms else "int8", share_of_bound=round(bound / t, 3))
            passes[v] = entry
            print(json.dumps(dict(log2_entries=lg, V=v, **entry)), flush=True)
        # ---- answer_many with the selection in place
        c1 = out["h1_squished"].shape[1]
        counts = [int(x) for x in a.counts.split(",")]
        qs = [[rng.integers(0, 2**32, 3 * cols, dtype=np.uint64).astype(np.uint32),
               rng.integers(0, 2**32, 3 * c1, dtype=np.uint64).astype(np.uint32)] for _ in range(max(counts))]
        srv = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, 1 << lg, 1, max_queries=max(counts))
        reqs = [D.serialize_request([q]) for q in qs]
        alone = [srv.answer(r) for r in reqs]
        many = {}
        identical = True
        for cnt in counts:
            got = srv.answer_many(reqs[:cnt])
            identical = identical and got == alone[:cnt]
            ms = median_ms(lambda: srv.answer_many(reqs[:cnt]), max(5, a.reps))
            many[cnt] = dict(call_ms=round(ms, 3), requests_per_s=round(cnt / ms * 1e3, 1))
        prof = {}
        try:
            ks = kernel_times(lambda: srv.answer_many(reqs[:64]))
            for nm, ms in ks:
                hit = re.search(r"k_\w+", nm)
                short = hit.group(0) if hit else nm.strip() or "?"
                p = prof.setdefault(short, dict(launches=0, ms=0.0))
                p["launches"] += 1
                p["ms"] = round(p["ms"] + ms, 4)
        except Exception as e:                                                    # the timings above stand on their own
            prof["error"] = repr(e)
        srv.close()
        dbm.close()
        res["sizes"].append(dict(log2_entries=lg, l=l, packed_cols=cols, db_mb=round(db_bytes / 1e6, 1), passes=passes,
                                 answer_many=many, answer_many_identical_to_alone=bool(identical), call64_kernels=prof))
        print(json.dumps(res["sizes"][-1]), flush=True)
    line = json.dumps(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
