"""DoublePIR over row shards: what sharding costs, and that the one-device path is unchanged.

  one   At 2^24 one-bit entries, kernel launches (b200pir_kernel_launches) per load, per answer() of one request and per
        answer_many of 64; at 2^33 entries, answer() latency (1 request) and answer_many throughput (64 requests).  With
        --parent DIR (a built checkout of the parent commit) the parent's and this tree's libraries run alternately, each
        in its own process, --rounds times, so the spread between rounds is measured beside the difference.
  shard At 2^36 entries, G = 1, 2 and 4 shards all on device 0 (after an untimed load that loads the modules): load time,
        answer latency, answer_many throughput at 64 requests, and the device time of the sharded path's extra work in one
        64-request call (torch.profiler, a run of its own): the sum kernel, and the copies by kind (each shard's msg[0]
        partials, device to device; the shards' partial responses to the first shard's device, peer or local).
  multi The sizes of --multi-sizes (default 2^38 and 2^39) on the devices of --multi-devices (default 0,1), each size below
        2^39 also on the first device alone.  The database is a seeded file (written to a temporary directory, as the tests
        write theirs) loaded with load_file_sharded.  Per layout: load time, per-device peak of device memory in use during
        the load (a side thread polls cudaMemGetInfo every 10 ms) and resident after it, answer latency, throughput at 64
        requests, and sampled responses decoded by the numpy client against the file's bits; where a size runs on both
        layouts, their responses are compared byte for byte.  Checks disk and host memory first (the decode holds A_1 and
        A_2 with their float halves, about 13 GB at 2^39) and reports "not measured" with the numbers when either is
        short, or when fewer GPUs are visible than the layout names.  --multi-devices 0,0 --multi-sizes 36 rehearses the
        same path on one GPU.

Latency: median wall clock of --reps calls that each synchronise, after a warm-up call.  Prints one JSON line with the card's
name and power limit, and writes it to --out if given.  Needs a GPU.

    python scripts/dpir_shard_probe.py [--parent DIR] [--rounds 2] [--reps 20] [--parts one,shard,multi]
                                       [--multi-devices 0,1] [--multi-sizes 38,39] [--out result.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


GIB = 1 << 30


def tests_module(name):
    """a helper module of tests/ (pick_params, the numpy client, the seeded-file writer)"""
    sys.path.insert(0, os.path.join(HERE, "tests"))
    return __import__(name)


def params(lg):
    """pick_params' shape for 2^lg one-bit entries (tests/test_oracle_doublepir_e2e.pick_params), the shape DESIGN names"""
    E = tests_module("test_oracle_doublepir_e2e")
    prm = E.pick_params(1 << lg, 1, E.SEC_PARAM, E.LOGQ)
    return {k: prm[k] for k in ("n", "l", "m", "logq", "p")}


def requests(D, prm, info, k, rng):
    dcols, c1 = (prm["m"] + 2) // 3, (prm["l"] // info["x"] + 2) // 3
    return [D.serialize_request([[rng.integers(0, 1 << 32, 3 * dcols, dtype=np.uint64).astype(np.uint32),
                                  rng.integers(0, 1 << 32, 3 * c1, dtype=np.uint64).astype(np.uint32)]]) for _ in range(k)]


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def serve_times(D, srv, prm, info, reps, rng):
    one = requests(D, prm, info, 1, rng)[0]
    many = requests(D, prm, info, 64, rng)
    lat = timed(lambda: srv.answer(one), reps)
    thr = timed(lambda: srv.answer_many(many), max(3, reps // 4))
    return dict(answer_ms=round(lat[0] * 1e3, 3), answer_ms_min_max=[round(lat[1] * 1e3, 3), round(lat[2] * 1e3, 3)],
                many64_per_s=round(64 / thr[0], 1), many64_ms_min_max=[round(thr[1] * 1e3, 3), round(thr[2] * 1e3, 3)])


def worker_one(reps):
    """the one-device path in whatever tree sdk_b200 is imported from"""
    import torch
    torch.cuda.init()
    import sdk_b200.doublepir as D
    from sdk_b200._lib import LIB
    out = {}
    rng = np.random.default_rng(1)
    for lg in (24, 33):
        prm = params(lg)
        num_entries = 1 << lg
        data = np.random.default_rng(lg).integers(0, 256, num_entries // 8, dtype=np.uint8)
        dbm, o, info = D.load(prm, num_entries, 1, data, D.ENTRY_BITS)        # modules loaded
        dbm.close()
        k0 = LIB.b200pir_kernel_launches()
        t0 = time.perf_counter()
        dbm, o, info = D.load(prm, num_entries, 1, data, D.ENTRY_BITS)
        load_s = time.perf_counter() - t0
        k_load = LIB.b200pir_kernel_launches() - k0
        srv = D.Server(dbm, o["h1_squished"], o["a2_t"], prm, num_entries, 1, max_queries=64)
        if lg == 24:
            one, many = requests(D, prm, info, 1, rng)[0], requests(D, prm, info, 64, rng)
            srv.answer(one)
            srv.answer_many(many)
            k0 = LIB.b200pir_kernel_launches()
            srv.answer(one)
            k1 = LIB.b200pir_kernel_launches()
            srv.answer_many(many)
            k2 = LIB.b200pir_kernel_launches()
            out["launches_2^24"] = dict(load=k_load, answer=k1 - k0, answer_many64=k2 - k1)
        else:
            out["times_2^33"] = dict(load_s=round(load_s, 3), **serve_times(D, srv, prm, info, reps, rng))
        srv.close()
        dbm.close()
    return out


def worker_shard(reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    import sdk_b200.doublepir as D
    lg = 36
    prm = params(lg)
    num_entries = 1 << lg
    data = np.frombuffer(np.random.default_rng(lg).bytes(num_entries // 8), dtype=np.uint8)
    out = dict(shape=prm)
    rng = np.random.default_rng(2)
    mats, _, _ = D.load_sharded(prm, num_entries, 1, data, [0], D.ENTRY_BITS)      # untimed: loads the modules
    for m in mats:
        m.close()
    for G in (1, 2, 4):
        t0 = time.perf_counter()
        mats, o, info = D.load_sharded(prm, num_entries, 1, data, [0] * G, D.ENTRY_BITS)
        load_s = time.perf_counter() - t0
        srv = D.Server(mats, o["h1_squished"], o["a2_t"], prm, num_entries, 1, max_queries=64)
        row = dict(load_s=round(load_s, 3), **serve_times(D, srv, prm, info, reps, rng))
        if G > 1:
            many = requests(D, prm, info, 64, rng)
            srv.answer_many(many)
            with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                srv.answer_many(many)
                torch.cuda.synchronize()
            ev = [(e.name, e.device_time_total / 1e3) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            row["many64_sum_kernel_ms"] = round(sum(t for n, t in ev if "k_dpir_sum_be" in n), 3)
            copies = {}
            for n, t in ev:
                if "Memcpy" in n and ("PtoP" in n or "DtoD" in n):
                    c = copies.setdefault(n.strip(), dict(count=0, ms=0.0))
                    c["count"] += 1
                    c["ms"] = round(c["ms"] + t, 3)
            row["many64_sharded_copies"] = copies       # DtoD: G x 64 msg[0] partials (and local shard copies); PtoP: G - 1
        out["G=%d" % G] = row
        srv.close()
        for m in mats:
            m.close()
    return out


class PeakPoller:
    """the most device memory in use on each device while the block runs, polled with cudaMemGetInfo on a side thread"""

    def __init__(self, devices, period=0.01):
        import torch
        self.torch, self.devices, self.period = torch, sorted(set(devices)), period
        self.free0 = {d: torch.cuda.mem_get_info(d)[0] for d in self.devices}
        self.low = dict(self.free0)
        self.stop = threading.Event()

    def _run(self):
        while not self.stop.is_set():
            for d in self.devices:
                self.low[d] = min(self.low[d], self.torch.cuda.mem_get_info(d)[0])
            self.stop.wait(self.period)

    def __enter__(self):
        self.th = threading.Thread(target=self._run, daemon=True)
        self.th.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.th.join()

    def peak_gb(self):
        return {d: round((self.free0[d] - self.low[d]) / 1e9, 1) for d in self.devices}

    def resident_gb(self):
        return {d: round((self.free0[d] - self.torch.cuda.mem_get_info(d)[0]) / 1e9, 1) for d in self.devices}


def decode_samples(D, prm, info, srv, h2, num_entries, bit, rng, edges, count=12):
    """answer_many of `count` single-query requests (file bits at indices 0, the last, the shard edges and random ones) decoded
    by the numpy client: (all decoded == file bits, the responses, the indices)"""
    E = tests_module("test_oracle_doublepir_e2e")
    LB = tests_module("test_gpu_dpir_load_bands")
    S = tests_module("test_gpu_dpir_serve")
    n, m, l = prm["n"], prm["m"], prm["l"]
    info = dict(info, bits=1)
    a_1 = D.derive_from_seed(m, n, D.SEED_A1)
    a_2 = D.derive_from_seed(l // info["x"], n, D.SEED_A2)
    a_2_sums = (a_2.astype(np.uint64).sum(axis=0) & np.uint64(0xFFFFFFFF)).reshape(1, n)   # all recover() reads of a_2
    mat_vec, E.mat_vec = E.mat_vec, LB._mat_vec_exact
    try:
        idxs = [0, num_entries - 1] + [e for e in edges if e < num_entries]
        idxs += [int(v) for v in rng.integers(0, num_entries, max(0, count - len(idxs)))]
        qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
        many = srv.answer_many([D.serialize_request([q]) for _, q in qs])
        ok = all(E.recover(i, h2, qmsg, S.flat(r), a_2_sums, client, prm, info) == bit(i)
                 for i, (client, qmsg), r in zip(idxs, qs, many))
    finally:
        E.mat_vec = mat_vec
        LB._halves.clear()
    return ok, many, idxs, qs


def worker_multi(reps, devices, sizes):
    import torch
    torch.cuda.init()
    visible = torch.cuda.device_count()
    if visible <= max(devices):
        return "not measured: %d GPU visible, the layout %s needs %d" % (visible, devices, max(devices) + 1)
    import sdk_b200.doublepir as D
    LB = tests_module("test_gpu_dpir_load_bands")
    out = {}
    rng = np.random.default_rng(3)
    for lg in sizes:
        prm = params(lg)
        num_entries = 1 << lg
        n, m = prm["n"], prm["m"]
        nbytes = num_entries // 8
        layouts = [[devices[0]], list(devices)] if lg < 39 else [list(devices)]
        tmp = tempfile.mkdtemp(prefix="dpir_shard_probe_")
        try:
            free_disk = shutil.disk_usage(tmp).free
            need_host = 6 * m * n * 8 + 2 * GIB
            if free_disk < nbytes + GIB:
                out["2^%d" % lg] = "not measured: disk %.1f GiB free in %s, %.1f GiB needed" % (free_disk / GIB, tmp, (nbytes + GIB) / GIB)
                continue
            if LB._mem_available() < need_host:
                out["2^%d" % lg] = "not measured: host memory %.1f GiB available, %.1f GiB needed to decode" % (
                    LB._mem_available() / GIB, need_host / GIB)
                continue
            path = os.path.join(tmp, "db.bin")
            t0 = time.perf_counter()
            LB._write_seeded(path, nbytes, lg)
            write_s = time.perf_counter() - t0
            fd = os.open(path, os.O_RDONLY)
            bit = lambda i: (os.pread(fd, 1, i >> 3)[0] >> (i & 7)) & 1
            first = None
            try:
                for devs in layouts:
                    key = "2^%d on %s" % (lg, devs)
                    torch.cuda.empty_cache()
                    try:
                        with PeakPoller(devs) as poll:
                            t0 = time.perf_counter()
                            mats, o, info = D.load_file_sharded(prm, num_entries, 1, path, devs, D.ENTRY_BITS)
                            load_s = time.perf_counter() - t0
                    except D.B200PirError as e:
                        out[key] = "not measured: %s" % e
                        continue
                    row = dict(shape=prm, file_write_s=round(write_s, 1), load_s=round(load_s, 3), peak_gb=poll.peak_gb(),
                               resident_gb=poll.resident_gb())
                    srv = D.Server(mats, o["h1_squished"], o["a2_t"], prm, num_entries, 1, max_queries=64)
                    try:
                        row.update(serve_times(D, srv, prm, info, reps, rng))
                        # the same samples on every layout (the multi-device layout's shard edges), so responses compare
                        edges = [r0 * prm["m"] * info["packing"] for r0, _ in D.shard_rows(prm, num_entries, 1, len(devices))[1:]]
                        ok, many, idxs, qs = decode_samples(D, prm, info, srv, o["h2"], num_entries, bit, np.random.default_rng(lg), edges)
                        row["decoded"] = dict(samples=len(idxs), all_equal_file_bits=bool(ok))
                        if first is None:
                            first = many
                        else:
                            row["responses_equal_first_layout"] = many == first
                    finally:
                        srv.close()
                        for mm in mats:
                            mm.close()
                    out[key] = row
            finally:
                os.close(fd)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    return out


def run_worker(tree, part, reps, extra=()):
    env = dict(os.environ, PYTHONPATH=tree)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", part, "--reps", str(reps)] + list(extra), cwd=tree,
                       env=env, capture_output=True, text=True)
    if r.returncode:
        return "failed: " + r.stderr.strip().splitlines()[-1] if r.stderr.strip() else "failed"
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--parts", default="one,shard,multi")
    ap.add_argument("--multi-devices", default="0,1")
    ap.add_argument("--multi-sizes", default="38,39")
    ap.add_argument("--worker")
    ap.add_argument("--out")
    a = ap.parse_args()
    if a.worker:
        sys.path.insert(0, os.getcwd())
        devices = [int(d) for d in a.multi_devices.split(",")]
        sizes = [int(v) for v in a.multi_sizes.split(",")]
        work = dict(one=worker_one, shard=worker_shard, multi=lambda r: worker_multi(r, devices, sizes))[a.worker]
        print(json.dumps(work(a.reps)))
        return
    res = dict(card=card())
    parts = a.parts.split(",")
    if "one" in parts:
        trees = [("parent", os.path.abspath(a.parent)), ("branch", HERE)] if a.parent else [("branch", HERE)]
        res["one"] = []
        for rnd in range(a.rounds):
            for name, tree in trees:
                res["one"].append(dict(tree=name, round=rnd, **{"result": run_worker(tree, "one", a.reps)}))
    for part in ("shard", "multi"):
        if part in parts:
            res[part] = run_worker(HERE, part, a.reps, ["--multi-devices", a.multi_devices, "--multi-sizes", a.multi_sizes])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
