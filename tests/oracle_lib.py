"""ctypes loader for the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (sdk_b200) never does.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(_ROOT, "oracle", "liboracle.so")

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)
u8p = C.POINTER(C.c_uint8)


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(_ROOT, "oracle")])


def _load():
    if not os.path.exists(_SO):
        build()
    lib = C.CDLL(_SO)
    lib.orc_last_error.restype = C.c_char_p
    lib.orc_params_new.restype = C.c_void_p
    lib.orc_params_new.argtypes = [C.c_uint64] * 12 + [C.c_int]
    lib.orc_params_new_raw.restype = C.c_void_p
    lib.orc_params_new_raw.argtypes = [C.c_uint64, u64p, C.c_uint64]
    lib.orc_params_free.argtypes = [C.c_void_p]
    lib.orc_client_new.restype = C.c_void_p
    lib.orc_client_new.argtypes = [C.c_void_p, C.c_uint64]
    lib.orc_client_free.argtypes = [C.c_void_p]
    for name in ("orc_get_bits_per", "orc_barrett_reduction_u128_raw", "orc_barrett_raw_u64", "orc_div2_uint_mod",
                 "orc_calc_index", "orc_rescale", "orc_recenter_mod", "orc_min_primitive_root", "orc_invert_uint_mod",
                 "orc_read_bits", "orc_splitmix64_at"):
        getattr(lib, name).restype = C.c_uint64
    lib.orc_get_bits_per.argtypes = [C.c_void_p, C.c_size_t]
    lib.orc_barrett_reduction_u128_raw.argtypes = [C.c_uint64] * 5
    lib.orc_barrett_raw_u64.argtypes = [C.c_uint64] * 3
    lib.orc_div2_uint_mod.argtypes = [C.c_uint64] * 2
    lib.orc_calc_index.argtypes = [u64p, u64p, C.c_uint64]
    lib.orc_rescale.argtypes = [C.c_uint64] * 3
    lib.orc_recenter_mod.argtypes = [C.c_uint64] * 3
    lib.orc_min_primitive_root.argtypes = [C.c_uint64] * 2
    lib.orc_invert_uint_mod.argtypes = [C.c_uint64] * 2
    lib.orc_splitmix64_at.argtypes = [C.c_uint64] * 2
    lib.orc_read_bits.argtypes = [u8p, C.c_size_t, C.c_size_t]
    lib.orc_write_bits.argtypes = [u8p, C.c_uint64, C.c_size_t, C.c_size_t]
    lib.orc_q2_value.restype = C.c_uint64
    lib.orc_q2_value.argtypes = [C.c_size_t]
    lib.orc_response_bytes.restype = C.c_size_t
    lib.orc_response_bytes.argtypes = [C.c_void_p]
    lib.orc_time_multiply.restype = C.c_double
    return lib


LIB = _load()


def _p64(a):
    if a is None:
        return None
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u64p)


def _p32(a):
    assert a.dtype == np.uint32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u32p)


def _p8(a):
    assert a.dtype == np.uint8 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u8p)


def _ck(rc):
    if rc != 0:
        raise RuntimeError("oracle: " + LIB.orc_last_error().decode())


PARAM_SETS = {
    # util.rs:122-137 get_fast_expansion_testing_params
    "T": dict(n=2, nu_1=6, nu_2=2, p=256, q2_bits=20, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
              db_item_size=8192, version=0),
    # version-1 packing, small (E1-shaped: t_gsw 7, t_conv 3, t_exp 5/5, instances 2)
    "T1": dict(n=2, nu_1=6, nu_2=2, p=256, q2_bits=22, t_gsw=7, t_conv=3, t_exp_left=5, t_exp_right=5, instances=2,
               db_item_size=16384, version=1),
    # distinct left/right expansion gadget (E0-shaped: t_exp 8/56, n=3)
    "T0": dict(n=3, nu_1=5, nu_2=3, p=256, q2_bits=20, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=56, instances=1,
               db_item_size=18432, version=0),
    # e2e-tests/params/v0.json
    "E0": dict(n=4, nu_1=9, nu_2=5, p=256, q2_bits=20, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=56, instances=1,
               db_item_size=32768, version=0),
    # e2e-tests/params/v1.json
    "E1": dict(n=2, nu_1=9, nu_2=5, p=256, q2_bits=22, t_gsw=7, t_conv=3, t_exp_left=5, t_exp_right=5, instances=4,
               db_item_size=32768, version=1),
    # SURVEY §8: S1 (1 GiB HBM-resident), S8 (1 GiB plaintext = 8 GiB HBM-resident)
    "S1": dict(n=2, nu_1=9, nu_2=5, p=256, q2_bits=22, t_gsw=7, t_conv=3, t_exp_left=5, t_exp_right=5, instances=1,
               db_item_size=8192, version=1),
    "S8": dict(n=2, nu_1=9, nu_2=8, p=256, q2_bits=22, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
               db_item_size=8192, version=0),
}


class Params:
    def __init__(self, expand_queries=True, **kw):
        self.kw = dict(kw)
        self.expand_queries = expand_queries
        order = ["n", "nu_1", "nu_2", "p", "q2_bits", "t_gsw", "t_conv", "t_exp_left", "t_exp_right", "instances",
                 "db_item_size", "version"]
        self.h = LIB.orc_params_new(*[int(kw[k]) for k in order], 1 if expand_queries else 0)
        if not self.h:
            raise RuntimeError(LIB.orc_last_error().decode())
        for k in order:
            setattr(self, k, int(kw[k]))
        info = np.zeros(32, dtype=np.uint64)
        _ck(LIB.orc_params_info(C.c_void_p(self.h), _p64(info)))
        names = ["poly_len", "crt_count", "q0", "q1", "modulus", "modulus_log2", "cr0_0", "cr1_0", "cr0_1", "cr1_1",
                 "cr0_mod", "cr1_mod", "mod0_inv_mod1", "mod1_inv_mod0", "g", "stop_round", "setup_bytes",
                 "query_bytes", "bytes_per_chunk", "modp_words_per_chunk"]
        for i, nm in enumerate(names):
            setattr(self, nm, int(info[i]))
        self.dim0 = 1 << self.nu_1
        self.num_per = 1 << self.nu_2
        self.trials = self.n * self.n
        self.slices = self.instances * self.trials
        self.N = self.poly_len
        self.W = self.crt_count * self.poly_len
        self.num_packing = self.n if self.version == 0 else 2
        self.has_right = expand_queries and (self.version == 0 or self.t_exp_right != self.t_exp_left)
        self.q2 = int(LIB.orc_q2_value(self.q2_bits))

    @staticmethod
    def named(name, **over):
        kw = dict(PARAM_SETS[name])
        eq = over.pop("expand_queries", True)
        kw.update(over)
        return Params(expand_queries=eq, **kw)

    @property
    def hp(self):
        return C.c_void_p(self.h)

    def __del__(self):
        try:
            LIB.orc_params_free(C.c_void_p(self.h))
        except Exception:
            pass

    # ---- primitives
    def ntt_table(self, mod, which):
        out = np.zeros(self.N, dtype=np.uint64)
        _ck(LIB.orc_ntt_table(self.hp, mod, which, _p64(out)))
        return out

    def ntt_forward(self, data):
        d = np.ascontiguousarray(data, dtype=np.uint64).copy()
        _ck(LIB.orc_ntt_forward(self.hp, _p64(d), C.c_size_t(d.size // self.W)))
        return d

    def ntt_inverse(self, data):
        d = np.ascontiguousarray(data, dtype=np.uint64).copy()
        _ck(LIB.orc_ntt_inverse(self.hp, _p64(d), C.c_size_t(d.size // self.W)))
        return d

    def to_ntt(self, raw, no_reduce=False):
        raw = np.ascontiguousarray(raw, dtype=np.uint64)
        npolys = raw.size // self.N
        out = np.zeros(npolys * self.W, dtype=np.uint64)
        _ck(LIB.orc_to_ntt(self.hp, _p64(out), _p64(raw), C.c_size_t(npolys), 1 if no_reduce else 0))
        return out

    def from_ntt(self, ntt):
        ntt = np.ascontiguousarray(ntt, dtype=np.uint64)
        npolys = ntt.size // self.W
        out = np.zeros(npolys * self.N, dtype=np.uint64)
        _ck(LIB.orc_from_ntt(self.hp, _p64(out), _p64(ntt), C.c_size_t(npolys)))
        return out

    def multiply(self, a, b, ar, ac, bc):
        out = np.zeros(ar * bc * self.W, dtype=np.uint64)
        _ck(LIB.orc_multiply(self.hp, _p64(out), _p64(a), _p64(b), C.c_size_t(ar), C.c_size_t(ac), C.c_size_t(bc)))
        return out

    def gadget_invert(self, inp, in_rows, in_cols, out_rows, rdim=None):
        out = np.zeros(out_rows * in_cols * self.N, dtype=np.uint64)
        _ck(LIB.orc_gadget_invert(self.hp, _p64(out), _p64(inp), C.c_size_t(in_rows), C.c_size_t(in_cols),
                                  C.c_size_t(out_rows), C.c_size_t(in_rows if rdim is None else rdim)))
        return out

    def build_gadget(self, rows, cols):
        out = np.zeros(rows * cols * self.N, dtype=np.uint64)
        _ck(LIB.orc_build_gadget(self.hp, _p64(out), C.c_size_t(rows), C.c_size_t(cols)))
        return out

    def bits_per(self, dim):
        return int(LIB.orc_get_bits_per(self.hp, dim))

    def automorph(self, inp, rows, t):
        out = np.zeros(rows * self.N, dtype=np.uint64)
        _ck(LIB.orc_automorph(self.hp, _p64(out), _p64(inp), C.c_size_t(rows), C.c_size_t(t)))
        return out

    # ---- stages
    def multiply_reg_by_database(self, db_slice, v_firstdim, dim0=None, num_per=None):
        dim0 = dim0 or self.dim0
        num_per = num_per or self.num_per
        out = np.zeros(num_per * 4 * self.N, dtype=np.uint64)
        _ck(LIB.orc_multiply_reg_by_database_shape(self.hp, _p64(out), _p64(db_slice), _p64(v_firstdim),
                                                   C.c_size_t(dim0), C.c_size_t(num_per)))
        return out

    def fold_ciphertexts(self, v_cts, v_folding, v_folding_neg, sparse=False):
        d = np.ascontiguousarray(v_cts, dtype=np.uint64).copy()
        num = d.size // (2 * self.N)
        _ck(LIB.orc_fold_ciphertexts(self.hp, _p64(d), C.c_size_t(num), _p64(v_folding), _p64(v_folding_neg),
                                     1 if sparse else 0))
        return d

    def get_v_folding_neg(self, v_folding):
        out = np.zeros_like(v_folding)
        _ck(LIB.orc_get_v_folding_neg(self.hp, _p64(out), _p64(v_folding)))
        return out

    def expand_query(self, pp, query_ct):
        vreg = np.zeros(self.dim0 * 2 * self.N, dtype=np.uint64)
        vf = np.zeros(self.nu_2 * 2 * 2 * self.t_gsw * self.W, dtype=np.uint64)
        _ck(LIB.orc_expand_query(self.hp, _p64(pp["left"]), _p64(pp["right"]), _p64(pp["conv"]), _p64(query_ct),
                                 _p64(vreg), _p64(vf)))
        return vreg, vf

    def coefficient_expansion(self, v, pp):
        d = np.ascontiguousarray(v, dtype=np.uint64).copy()
        _ck(LIB.orc_coefficient_expansion(self.hp, _p64(d), _p64(pp["left"]), _p64(pp["right"])))
        return d

    def regev_to_gsw(self, v_inp, conv):
        n_inp = v_inp.size // (2 * self.W)
        out = np.zeros((n_inp // self.t_gsw) * 2 * 2 * self.t_gsw * self.W, dtype=np.uint64)
        _ck(LIB.orc_regev_to_gsw(self.hp, _p64(out), _p64(v_inp), C.c_size_t(n_inp), _p64(conv)))
        return out

    def pack(self, v_ct, v_packing):
        out = np.zeros((self.n + 1) * self.n * self.W, dtype=np.uint64)
        _ck(LIB.orc_pack(self.hp, _p64(out), _p64(v_ct), _p64(v_packing)))
        return out

    def response_bytes(self):
        return int(LIB.orc_response_bytes(self.hp))

    def encode(self, packed_raw):
        out = np.zeros(self.response_bytes() + 16, dtype=np.uint8)
        ln = C.c_size_t(0)
        _ck(LIB.orc_encode(self.hp, _p8(out), C.byref(ln), _p64(packed_raw)))
        return out[: ln.value].copy()

    def process_query(self, pp, query, db, dump=False, sparse_fold=False):
        """query: dict(ct=...) or dict(v_buf=..., v_ct=...).  sparse_fold: fold like lib/server (compute/fold.rs:15-65)."""
        LIB.orc_set_sparse_fold(1 if sparse_fold else 0)
        try:
            return self._process_query(pp, query, db, dump)
        finally:
            LIB.orc_set_sparse_fold(0)

    def _process_query(self, pp, query, db, dump=False):
        out = np.zeros(self.response_bytes() + 16, dtype=np.uint8)
        ln = C.c_size_t(0)
        d = {}
        if dump:
            d["v_firstdim"] = np.zeros(self.dim0 * 2 * self.N, dtype=np.uint64)
            d["v_folding"] = np.zeros(self.nu_2 * 4 * self.t_gsw * self.W, dtype=np.uint64)
            d["v_folding_neg"] = np.zeros(self.nu_2 * 4 * self.t_gsw * self.W, dtype=np.uint64)
            d["first_mult"] = np.zeros(self.num_per * 4 * self.N, dtype=np.uint64)
            d["folded"] = np.zeros(self.slices * 2 * self.N, dtype=np.uint64)
            d["packed"] = np.zeros(self.instances * (self.n + 1) * self.n * self.N, dtype=np.uint64)
        g = lambda k: _p64(d[k]) if dump else None
        _ck(LIB.orc_process_query(self.hp, _p64(pp["pack"]), _p64(pp.get("left")), _p64(pp.get("right")),
                                  _p64(pp.get("conv")), _p64(query.get("ct")), _p64(query.get("v_buf")),
                                  _p64(query.get("v_ct")), _p64(db), _p8(out), C.byref(ln), g("v_firstdim"),
                                  g("v_folding"), g("v_folding_neg"), g("first_mult"), g("folded"), g("packed")))
        resp = out[: ln.value].copy()
        return (resp, d) if dump else resp

    def pp_deserialize(self, data):
        sz = np.zeros(4, dtype=np.uint64)
        _ck(LIB.orc_pp_sizes(self.hp, _p64(sz)))
        sz[0] = self.n * (self.n + 1) * self.t_conv * self.W            # deserialize always builds params.n packing matrices
        arrs = [np.zeros(int(x), dtype=np.uint64) if x else None for x in sz]
        data = np.ascontiguousarray(data, dtype=np.uint8)
        _ck(LIB.orc_pp_deserialize(self.hp, _p8(data), C.c_size_t(data.size), *[_p64(a) for a in arrs]))
        return dict(pack=arrs[0], left=arrs[1], right=arrs[2], conv=arrs[3])

    def query_deserialize(self, data):
        ct = np.zeros(2 * self.N, dtype=np.uint64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        _ck(LIB.orc_query_deserialize(self.hp, _p8(data), C.c_size_t(data.size), _p64(ct)))
        return ct

    def query_deserialize_direct(self, data):
        """Query::deserialize, direct-upload branch (client.rs:316-327): -> dict(v_buf, v_ct)."""
        v_buf = np.zeros(self.dim0 * 2 * self.N, dtype=np.uint64)
        v_ct = np.zeros(self.nu_2 * 2 * 2 * self.t_gsw * self.N, dtype=np.uint64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        _ck(LIB.orc_query_deserialize_direct(self.hp, _p8(data), C.c_size_t(data.size), _p64(v_buf), _p64(v_ct)))
        return dict(v_buf=v_buf, v_ct=v_ct)

    def load_db_from_bytes(self, data):
        """load_db_from_seek (server.rs:320-357) over an in-memory file image -> db words."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        db = np.zeros(self.slices * self.dim0 * self.num_per * self.N, dtype=np.uint64)
        _ck(LIB.orc_load_db_from_bytes(self.hp, _p8(data), C.c_size_t(data.size), _p64(db)))
        return db

    def generate_db(self, seed):
        db = np.zeros(self.slices * self.dim0 * self.num_per * self.N, dtype=np.uint64)
        _ck(LIB.orc_generate_db(self.hp, C.c_uint64(seed), _p64(db)))
        return db

    def update_item_raw(self, data):
        """lib/server db/loading.rs:317-359: bucket bytes -> [slices][2048] packed item polynomials."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        out = np.zeros(self.slices * self.N, dtype=np.uint64)
        _ck(LIB.orc_update_item_raw(self.hp, _p8(data), C.c_size_t(data.size), _p64(out)))
        return out

    def db_plain_item(self, seed, idx):
        out = np.zeros(self.instances * self.n * self.n * self.N, dtype=np.uint64)
        _ck(LIB.orc_db_plain_item(self.hp, C.c_uint64(seed), C.c_uint64(idx), _p64(out)))
        return out


class Client:
    def __init__(self, params, seed):
        self.p = params
        self.h = LIB.orc_client_new(params.hp, C.c_uint64(seed))

    def __del__(self):
        try:
            LIB.orc_client_free(C.c_void_p(self.h))
        except Exception:
            pass

    def generate_keys(self):
        sz = np.zeros(4, dtype=np.uint64)
        _ck(LIB.orc_pp_sizes(self.p.hp, _p64(sz)))
        arrs = [np.zeros(int(s), dtype=np.uint64) if s else None for s in sz]
        _ck(LIB.orc_client_generate_keys(C.c_void_p(self.h), *[_p64(a) for a in arrs]))
        return dict(pack=arrs[0], left=arrs[1], right=arrs[2], conv=arrs[3])

    def generate_query(self, idx):
        p = self.p
        if p.expand_queries:
            ct = np.zeros(2 * p.N, dtype=np.uint64)
            _ck(LIB.orc_client_generate_query(C.c_void_p(self.h), C.c_uint64(idx), _p64(ct), None, None))
            return dict(ct=ct)
        v_buf = np.zeros(p.dim0 * 2 * p.N, dtype=np.uint64)
        v_ct = np.zeros(p.nu_2 * 2 * 2 * p.t_gsw * p.N, dtype=np.uint64)
        _ck(LIB.orc_client_generate_query(C.c_void_p(self.h), C.c_uint64(idx), None, _p64(v_buf), _p64(v_ct)))
        return dict(v_buf=v_buf, v_ct=v_ct)

    def pp_bytes(self):
        """PublicParameters::serialize of the last generated keys (client.rs:198-210)."""
        out = np.zeros(self.p.setup_bytes + 64, dtype=np.uint8)
        n = C.c_size_t(0)
        _ck(LIB.orc_client_pp_bytes(C.c_void_p(self.h), _p8(out), C.byref(n)))
        return out[: n.value].copy()

    def query_bytes(self):
        """Query::serialize of the last generated query (client.rs:279-301)."""
        out = np.zeros(self.p.query_bytes + 64, dtype=np.uint8)
        n = C.c_size_t(0)
        _ck(LIB.orc_client_query_bytes(C.c_void_p(self.h), _p8(out), C.byref(n)))
        return out[: n.value].copy()

    def decode_response(self, resp):
        p = self.p
        out = np.zeros(p.instances * p.n * p.n * p.N, dtype=np.uint64)
        resp = np.ascontiguousarray(resp, dtype=np.uint8)
        _ck(LIB.orc_client_decode_response(C.c_void_p(self.h), _p8(resp), C.c_size_t(resp.size), _p64(out)))
        return out

    def decode_numerators(self, resp):
        """The numerators decode_response rounds (client.rs:780-800): int64, same layout as decode_response's output.
        Coefficient k decodes to round(numer[k] / denom) mod p with denom = q2 * (q1 / p) = q2 * 4."""
        p = self.p
        out = np.zeros(p.instances * p.n * p.n * p.N, dtype=np.int64)
        resp = np.ascontiguousarray(resp, dtype=np.uint8)
        _ck(LIB.orc_client_decode_numerators(C.c_void_p(self.h), _p8(resp), C.c_size_t(resp.size),
                                             out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def encrypt_reg(self, sigma_raw):
        out = np.zeros(2 * self.p.W, dtype=np.uint64)
        _ck(LIB.orc_client_encrypt_reg(C.c_void_p(self.h), _p64(np.ascontiguousarray(sigma_raw, dtype=np.uint64)), _p64(out)))
        return out

    def decrypt_reg(self, ct_ntt):
        out = np.zeros(self.p.N, dtype=np.uint64)
        _ck(LIB.orc_client_decrypt_reg(C.c_void_p(self.h), _p64(np.ascontiguousarray(ct_ntt, dtype=np.uint64)), _p64(out)))
        return out


def dpir_matvec_packed(a, b, rows, cols):
    out = np.zeros(rows, dtype=np.uint32)
    _ck(LIB.orc_dpir_matvec_packed(_p32(out), _p32(a), _p32(b), C.c_size_t(rows), C.c_size_t(cols)))
    return out


def dpir_mul(a, b, ar, ac, bc):
    """matrix/ops.rs:169-191 (wrapping u32): (ar x ac) * (ac x bc)."""
    out = np.zeros(ar * bc, dtype=np.uint32)
    _ck(LIB.orc_dpir_mul(_p32(out), _p32(np.ascontiguousarray(a, dtype=np.uint32)), _p32(np.ascontiguousarray(b, dtype=np.uint32)),
                         C.c_size_t(ar), C.c_size_t(ac), C.c_size_t(bc)))
    return out.reshape(ar, bc)


def dpir_setup(db, l, m, a1, n, a2, p, delta, x):
    """doublepir.rs:76-108.  db: l x m centered entries; a1: m x n; a2: (l/x) x n.  Returns dict(db_sq, h1_sq, a2_t, h2)."""
    rows1 = n * delta * x
    lx = l // x
    lx3 = lx + (3 - lx % 3) % 3
    out = dict(db_sq=np.zeros((l, (m + 2) // 3), dtype=np.uint32), h1_sq=np.zeros((rows1, (lx + 2) // 3), dtype=np.uint32),
               a2_t=np.zeros((n, lx3), dtype=np.uint32), h2=np.zeros((rows1, n), dtype=np.uint32))
    _ck(LIB.orc_dpir_setup(_p32(np.ascontiguousarray(db, dtype=np.uint32)), C.c_size_t(l), C.c_size_t(m),
                           _p32(np.ascontiguousarray(a1, dtype=np.uint32)), C.c_size_t(n),
                           _p32(np.ascontiguousarray(a2, dtype=np.uint32)), C.c_uint32(p), C.c_size_t(delta), C.c_size_t(x),
                           _p32(out["db_sq"]), _p32(out["h1_sq"]), _p32(out["a2_t"]), _p32(out["h2"])))
    return out


def dpir_matrix_mul_transposed_packed(a, b, a_rows, a_cols, b_rows, b_cols):
    out = np.zeros(a_rows * b_rows, dtype=np.uint32)
    _ck(LIB.orc_dpir_matrix_mul_transposed_packed(_p32(out), _p32(a), _p32(b), C.c_size_t(a_rows), C.c_size_t(a_cols),
                                                  C.c_size_t(b_rows), C.c_size_t(b_cols)))
    return out


def dpir_transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat):
    out_rows, out_cols = cols * delta * concat, (rows // concat + 2) // 3
    out = np.zeros(out_rows * out_cols, dtype=np.uint32)
    _ck(LIB.orc_dpir_transpose_expand_concat_cols_squish(_p32(out), _p32(a), C.c_size_t(rows), C.c_size_t(cols),
                                                         C.c_uint64(modulus), C.c_size_t(delta), C.c_size_t(concat)))
    return out, out_rows, out_cols


def dpir_answer(db, db_rows, db_cols, queries, h_1, h1_rows, h1_cols, a2t, a2t_rows, a2t_cols, p, delta, x, ne, chunk_idx=None):
    """doublepir.rs:246-350.  queries: list of [q_1, q_2...] uint32 arrays.  chunk_idx = k: the server that holds only the
    k-th batch of rows (raw_data = that slice, :268-275): the other batches contribute zero rows (:270-273)."""
    nq = len(queries)
    batch = db_rows // nq
    parts, last = [], 0
    for b, q in enumerate(queries):
        bs = db_rows - last if b == nq - 1 else batch
        if chunk_idx is not None and b != chunk_idx:
            parts.append(np.zeros(bs, dtype=np.uint32))
        else:
            parts.append(dpir_matvec_packed(np.ascontiguousarray(db[last * db_cols:(last + bs) * db_cols]), q[0], bs, db_cols))
        last += bs
    a_1 = np.concatenate(parts)
    a_1, r1, c1 = dpir_transpose_expand_concat_cols_squish(a_1, db_rows, 1, p, delta, x)
    msg = [dpir_matrix_mul_transposed_packed(a_1, a2t, r1, c1, a2t_rows, a2t_cols)]
    for q in queries:
        for j in range(ne // x):
            msg.append(dpir_matvec_packed(h_1, q[1 + j], h1_rows, h1_cols))
            msg.append(dpir_matvec_packed(a_1, q[1 + j], r1, c1))
    return msg
