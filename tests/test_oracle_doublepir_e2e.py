"""DoublePIR end to end on the CPU oracle, the way the reference's own test pins the scheme
(lib/doublepir/src/doublepir/doublepir.rs:469-525 simple_end_to_end_test): pick_params -> Db::with_data -> setup -> query ->
answer -> recover == the planted entry.  The server side (setup, answer) is the oracle's C++ restatement that the GPU kernels
are compared with bit for bit; the client side (query, recover) and the database packing are restated here in numpy — harness
only, each function citing the lines it follows.  The shared matrices A_1, A_2 are uniform (the reference derives them from
AES-128-CTR seeds, matrix/derivation.rs; any uniform matrix is a valid public parameter, and nothing on the server path
depends on how they were drawn)."""
import math

import numpy as np
import pytest

import oracle_lib as O

LOGQ, SEC_PARAM, COMP_RATIO, MAX_SEARCH_P = 32, 1 << 10, 64, 1 << 20          # doublepir.rs:5-15
PARAMS_STORE = [(10, 13, 32, 6.4, 9, 991, 929), (10, 14, 32, 6.4, 9, 833, 781), (10, 15, 32, 6.4, 9, 701, 657),
                (10, 16, 32, 6.4, 9, 589, 552), (10, 17, 32, 6.4, 8, 495, 464), (10, 18, 32, 6.4, 8, 416, 390),
                (10, 19, 32, 6.4, 8, 350, 328), (10, 20, 32, 6.4, 8, 294, 276), (10, 21, 32, 6.4, 7, 247, 231)]   # params_store.rs
Q = 1 << LOGQ
U32 = np.uint32


def num_db_entries(num_entries, bits, p):                                     # database.rs:356-374
    if bits <= math.log2(p):
        per_elem = int(math.log2(p)) // bits
        return math.ceil(num_entries / per_elem), 1, per_elem
    ne = math.ceil(bits / math.log2(p))
    return num_entries * ne, ne, 0


def approx_database_dims(num_entries, bits, p, lower_bound_m):                # database.rs:376-418
    db_elems, ne, _ = num_db_entries(num_entries, bits, p)
    l = int(math.floor(math.sqrt(db_elems)))
    if l % ne:
        l += ne - l % ne
    m = math.ceil(db_elems / l)
    if m >= lower_bound_m:
        return l, m
    m = lower_bound_m
    l = math.ceil(db_elems / m)
    if l % ne:
        l += ne - l % ne
    return l, m


def params_pick(n, logq, l, m, max_samples):                                  # params.rs:76-104
    for logn, logm, lq, sigma, _, _, p_double in PARAMS_STORE:
        if n == 1 << logn and max_samples <= 1 << logm and logq == lq:
            return dict(n=n, l=l, m=m, logq=logq, sigma=sigma, p=512 if p_double == 552 else p_double)
    raise AssertionError("No suitable params known!")


def pick_params(num_entries, bits, n, logq):                                  # doublepir.rs:17-43
    good, mod_p = None, 2
    while mod_p < MAX_SEARCH_P:
        l, m = approx_database_dims(num_entries, bits, mod_p, COMP_RATIO * n)
        p = params_pick(n, logq, l, m, max(l, m))
        if p["p"] < mod_p:
            assert good is not None
            return good
        good, mod_p = p, mod_p + 1
    raise AssertionError("Could not find params")


def base_p(p, m, i):                                                          # arith.rs:16-22
    return (m // p ** i) % p


def reconstruct_from_base_p(p, vals):                                         # arith.rs:1-13
    return sum(int(v) * p ** i for i, v in enumerate(vals))


def db_with_data(num_entries, bits, prm, data):                               # database.rs:56-90, :170-205
    db_elems, ne, packing = num_db_entries(num_entries, bits, prm["p"])
    assert db_elems <= prm["l"] * prm["m"]
    info = dict(num_entries=num_entries, bits=bits, packing=packing, ne=ne, x=ne, p=prm["p"], logq=prm["logq"])
    l, m = prm["l"], prm["m"]
    mat = np.zeros((l, m), dtype=np.uint64)
    if packing > 0:
        pad = (-len(data)) % packing
        d = np.concatenate([data.astype(np.uint64), np.zeros(pad, dtype=np.uint64)]).reshape(-1, packing)
        cur = np.zeros(d.shape[0], dtype=np.uint64)
        for k in range(packing):
            cur += d[:, k] << np.uint64(bits * k)
        mat.reshape(-1)[: cur.size] = cur
    else:
        i = np.arange(len(data))
        for j in range(ne):
            mat[(i // m) * ne + j, i % m] = (data.astype(np.uint64) // np.uint64(prm["p"] ** j)) % np.uint64(prm["p"])
    return info, (mat.astype(np.int64) - prm["p"] // 2).astype(np.uint32)        # "Map DB elems to [-p/2; p/2]"


def gaussian(rng, n):                                                         # matrix/gaussian.rs:4-10 (sigma 6.4, rounded)
    return np.round(rng.standard_normal(n) * 6.4).astype(np.int64).astype(np.uint32)


def mat_vec(a, v):                                                            # matrix/ops.rs:169-191, wrapping u32
    return (a.astype(np.uint64) @ v.astype(np.uint64)).astype(np.uint32)      # wraps mod 2^64, then the low 32 bits


# ---- the server's packed kernels, defined in numpy (uint64 sums masked to 32 bits) ---------------------------------------
def unpack_fields(a, rows, cols):                                            # kernels.rs:9-12: 3 x 10 bits a word, bits 30-31 unused
    w = np.asarray(a, dtype=np.uint64).reshape(rows, cols, 1)
    return ((w >> (np.uint64(10) * np.arange(3, dtype=np.uint64))) & np.uint64(1023)).reshape(rows, 3 * cols)


def np_matvec_packed(a, b, rows, cols):                                       # kernels.rs:14-178 matrix_mul_vec_packed
    return ((unpack_fields(a, rows, cols) @ b.astype(np.uint64)) & np.uint64(0xFFFFFFFF)).astype(U32)


def np_matrix_mul_transposed_packed(a, b, a_rows, a_cols, b_rows, b_cols):     # kernels.rs:180-278, both branches
    bm = b.astype(np.uint64).reshape(b_rows, b_cols)[:, : 3 * a_cols]
    return ((unpack_fields(a, a_rows, a_cols) @ bm.T) & np.uint64(0xFFFFFFFF)).astype(U32).reshape(-1)


def np_transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat):   # matrix/indexing.rs:117-143, basis 10, d 3
    out_rows, out_cols = cols * delta * concat, (rows // concat + 2) // 3
    out = np.zeros((out_rows, out_cols), dtype=np.uint64)
    val = np.asarray(a, dtype=np.uint64).reshape(rows, cols)
    j = np.arange(rows, dtype=np.uint64)[:, None]
    i = np.arange(cols, dtype=np.uint64)[None, :]
    c = j // np.uint64(concat)
    for f in range(delta):
        r = (i * np.uint64(delta) + np.uint64(f)) + np.uint64(cols * delta) * (j % np.uint64(concat))
        r, cd = np.broadcast_arrays(r, c // np.uint64(3))
        np.add.at(out, (r.astype(np.int64), cd.astype(np.int64)), (val % np.uint64(modulus)) << (np.uint64(10) * (c % np.uint64(3))))
        val //= np.uint64(modulus)
    return (out & np.uint64(0xFFFFFFFF)).astype(U32).reshape(-1), out_rows, out_cols


def query(i, a_1, a_2, prm, info, rng):                                       # doublepir.rs:111-160
    idx = i // info["packing"] if info["packing"] > 0 else i
    i1 = (idx // prm["m"]) * (info["ne"] // info["x"])
    i2 = idx % prm["m"]
    ext_delta = Q // prm["p"]
    secret1 = rng.integers(0, Q, prm["n"], dtype=np.uint64).astype(U32)       # random_logmod(n, 1, logq)
    query1 = mat_vec(a_1, secret1) + gaussian(rng, prm["m"])
    query1[i2] += U32(ext_delta)
    if prm["m"] % 3:
        query1 = np.concatenate([query1, np.zeros(3 - prm["m"] % 3, dtype=U32)])
    state, msg = [secret1], [query1]
    lx = prm["l"] // info["x"]
    for j in range(info["ne"] // info["x"]):
        secret2 = gaussian(rng, prm["n"])
        query2 = mat_vec(a_2, secret2) + gaussian(rng, lx)
        query2[i1 + j] += U32(ext_delta)
        if lx % 3:
            query2 = np.concatenate([query2, np.zeros(3 - lx % 3, dtype=U32)])
        state.append(secret2)
        msg.append(query2)
    return state, msg


def recover(i, offline_h2, qmsg, answer, a_2, client, prm, info, batch_index=0):   # doublepir.rs:352-458
    n, p, x, ne = prm["n"], prm["p"], info["x"], info["ne"]
    delta = math.ceil(prm["logq"] / math.log2(p))
    ext_delta = Q // p
    rnd = lambda v: ((v.astype(np.uint64) + np.uint64(ext_delta // 2)) // np.uint64(ext_delta)) % np.uint64(p)   # params.rs:26-28
    ratio = p // 2
    val1 = (Q - (ratio * int(qmsg[0][: prm["m"]].astype(np.uint64).sum())) % Q) % Q
    val2 = (Q - (ratio * int(qmsg[1][: prm["l"] // x].astype(np.uint64).sum())) % Q) % Q
    h1 = answer[0].reshape(delta * x, n).copy()
    val3 = (Q - (ratio * a_2.astype(np.uint64).sum(axis=0)) % Q) % Q                      # per column j1 of a_2
    h1 = (h1.astype(np.uint64) + val3[None, :]).astype(U32)
    secret1 = client[0]
    vals = []
    offset = (ne // x * 2) * batch_index                                       # "for batching"
    for k in range(ne // x):
        a2 = answer[1 + 2 * k + offset]
        h2 = (answer[2 + 2 * k + offset].astype(np.uint64) + val2).astype(U32)
        secret2 = client[1 + k]
        for j in range(x):
            state = np.concatenate([(a2[j * n * delta:(j + 1) * n * delta].astype(np.uint64) + val2).astype(U32),
                                    h2[j * delta:(j + 1) * delta]])
            hint = np.concatenate([offline_h2[j * n * delta:(j + 1) * n * delta], h1[j * delta:(j + 1) * delta]])
            state = state - mat_vec(hint, secret2)                             # wrapping u32
            state = rnd(state)                                                 # values in [0, p)
            # contract (matrix/contract.rs:37-56): delta values, centered -> raw, base-p digits of one 32-bit value
            raw = (state + np.uint64(p // 2)) % np.uint64(p)
            raw = raw.reshape(n + 1, delta)
            contracted = np.zeros(n + 1, dtype=np.uint64)
            for f in range(delta):
                contracted += raw[:, f] * np.uint64(p ** f)
            contracted = contracted.astype(U32)
            prod = (secret1.astype(np.uint64) * contracted[:n].astype(np.uint64)) & np.uint64(Q - 1)   # u32 wrapping products
            noised = (int(contracted[n]) + val1 - int(prod.sum())) % Q
            vals.append((noised + ext_delta // 2) // ext_delta % p)
    # Db::reconstruct_elem, database.rs:283-302
    vals = [((v + p // 2) % Q) % p for v in vals]
    val = reconstruct_from_base_p(p, vals)
    if info["packing"] > 0:
        val = base_p(1 << info["bits"], val, i % info["packing"])
    return val


_prepared = {}


def prepare(num_entries, bits, seed, full_width=False):
    """pick_params, Db::with_data, init, setup (cached: the 2^24-entry setup is shared by several tests).  full_width plants
    values of all `bits` bits instead of bytes, so that entries wider than 8 bits have non-zero high base-p digits."""
    full_width = full_width and bits > 8
    key = (num_entries, bits, seed, full_width)
    if key not in _prepared:
        rng = np.random.default_rng(seed)
        prm = pick_params(num_entries, bits, SEC_PARAM, LOGQ)
        if full_width:
            data = rng.integers(0, 1 << bits, num_entries, dtype=np.uint64)
        else:
            data = rng.integers(0, min(1 << bits, 256), num_entries, dtype=np.uint8)   # the reference's iterator yields u8 items
        info, db = db_with_data(num_entries, bits, prm, data)
        n, l, m, p, x = prm["n"], prm["l"], prm["m"], prm["p"], info["x"]
        delta = math.ceil(LOGQ / math.log2(p))
        a_1 = rng.integers(0, Q, (m, n), dtype=np.uint64).astype(U32)              # init(), doublepir.rs:46-51
        a_2 = rng.integers(0, Q, (l // x, n), dtype=np.uint64).astype(U32)
        st = O.dpir_setup(db, l, m, a_1, n, a_2, p, delta, x)                      # server_state = [h1_sq, a2_t], hint = [h2]
        _prepared[key] = (rng, prm, data, info, delta, a_1, a_2, st)
    return _prepared[key]


def run_answer(st, prm, info, delta, queries, chunk_idx=None):
    n, l, m, p, x, ne = prm["n"], prm["l"], prm["m"], prm["p"], info["x"], info["ne"]
    lx = l // x
    return O.dpir_answer(st["db_sq"].reshape(-1), l, (m + 2) // 3, queries, st["h1_sq"].reshape(-1), n * delta * x, (lx + 2) // 3,
                         st["a2_t"].reshape(-1), n, st["a2_t"].shape[1], p, delta, x, ne, chunk_idx=chunk_idx)


@pytest.mark.parametrize("num_entries,bits,seed", [(1 << 24, 1, 1), (1 << 20, 10, 2)])
def test_simple_end_to_end(num_entries, bits, seed):
    rng, prm, data, info, delta, a_1, a_2, st = prepare(num_entries, bits, seed)
    if bits == 1:
        assert (prm["l"], prm["m"], prm["p"]) == (29, 65536, 512)              # the shape SURVEY 8(d) quotes for this test
    for i in [0, num_entries - 1] + [int(v) for v in rng.integers(0, num_entries, 3)]:
        client, qmsg = query(i, a_1, a_2, prm, info, rng)
        ans = run_answer(st, prm, info, delta, [qmsg])
        assert len(ans) == 1 + 2 * (info["ne"] // info["x"])
        got = recover(i, st["h2"], qmsg, ans, a_2, client, prm, info)
        assert got == int(data[i]), (i, got, int(data[i]))


def test_batched_end_to_end():
    # doublepir.rs:526-606 batched_end_to_end_test: two queries in one answer(), each selecting a column from ITS batch of
    # rows (rows 0..13 and 14..28 of the 29); one shared h1, per-query (a_2, h_2) pairs at offset 2 * batch_index
    num_entries, bits = 1 << 24, 1
    rng, prm, data, info, delta, a_1, a_2, st = prepare(num_entries, bits, 1)
    batch_sz = 14 * 65536 * 9
    for _ in range(2):
        i1 = int(rng.integers(0, batch_sz))
        i2 = (i1 + batch_sz) % num_entries
        idxs = sorted([i1, i2])
        qs = [query(i, a_1, a_2, prm, info, rng) for i in idxs]
        ans = run_answer(st, prm, info, delta, [q for _, q in qs])
        assert len(ans) == 1 + 2 * 2
        for b, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
            assert recover(i, st["h2"], qmsg, ans, a_2, client, prm, info, batch_index=b) == int(data[i]), (b, i)


def test_chunked_end_to_end():
    # doublepir.rs:607-716 chunked_end_to_end_test: the database rows split over two servers, each answers from its slice
    # alone; the first message and every h_2 add up across servers, the a_2 messages are identical on both.  This is the
    # model for sharding DoublePIR over GPUs with no collective (DESIGN section 6).
    num_entries, bits = 1 << 24, 1
    rng, prm, data, info, delta, a_1, a_2, st = prepare(num_entries, bits, 1)
    batch_sz = 14 * 65536 * 9
    i1 = int(rng.integers(0, batch_sz))
    idxs = sorted([i1, (i1 + batch_sz) % num_entries])
    qs = [query(i, a_1, a_2, prm, info, rng) for i in idxs]
    full = None
    for chunk in range(2):
        resp = run_answer(st, prm, info, delta, [q for _, q in qs], chunk_idx=chunk)
        assert len(resp) == 1 + 2 * 2
        if full is None:
            full = [r.copy() for r in resp]
        else:
            for k in range(len(resp)):
                if k % 2 == 1:
                    assert np.array_equal(full[k], resp[k])        # a_2 = h_1 * q_2 does not depend on the rows held
                    continue
                full[k] = full[k] + resp[k]                        # wrapping u32
    whole = run_answer(st, prm, info, delta, [q for _, q in qs])
    for a, b in zip(full, whole):
        assert np.array_equal(a, b)                                # the per-server answers add up to the one-server answer
    for b, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
        assert recover(i, st["h2"], qmsg, full, a_2, client, prm, info, batch_index=b) == int(data[i]), (b, i)
