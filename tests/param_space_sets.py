"""Parameter sets that cover the corners of the space b200pir_ctx_create accepts (n 1..4, gadget dimensions 3..56, p up to 2^20,
q2_bits 14..36, nu_1 down to 1, version 1 with distinct left/right expansion gadgets, direct upload), beyond the named sets of
oracle_lib.PARAM_SETS.  Shared by test_oracle_param_space.py (the CPU oracle at these points) and test_gpu_param_space.py (the
CUDA path against the oracle).

Every set is written as overrides of BASE (the T set, util.rs:122-137).  `decodes` says whether the client recovers the
planted item at these parameters: the sets marked False are noise-limited (gadget width 4 everywhere, t_gsw = 3 with
expansion, p >= 2^16 with expansion), so the response bytes are still deterministic integer arithmetic and must match bit
for bit, but decoding them is not a property of the parameters."""

BASE = dict(n=2, nu_1=6, nu_2=2, p=256, q2_bits=20, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
            db_item_size=0, version=0)

# version-1 gadget shape of E1 / T1
_V1 = dict(version=1, t_gsw=7, t_conv=3, t_exp_left=5, t_exp_right=5, q2_bits=22)

# name -> (overrides of BASE, expand_queries, decodes)
SETS = {
    # spiral-rs util.rs CFG_16_100000 shrunk: t_gsw = 10 (20 products per fold accumulator: the mid-loop reduction), p = 512
    "cfg16_shrunk": (dict(t_gsw=10, t_conv=4, t_exp_left=16, t_exp_right=56, p=512, q2_bits=21, instances=3, nu_2=3), True, True),
    # lib/server compute/dot_product.rs tests: t_gsw = 9 (odd: the fold's lone last digit) on version 1
    "tgsw9_v1": (dict(_V1, t_gsw=9), True, True),
    # spiral-rs client.rs default parameters (the only large set: 512 x 64 items)
    "client_default": (dict(nu_1=9, nu_2=6, t_gsw=10, t_conv=4, t_exp_left=16, t_exp_right=56), True, True),
    "n1": (dict(n=1), True, True),
    "n1_nu2_0": (dict(n=1, nu_2=0), True, True),
    "n1_nu1_10": (dict(n=1, nu_1=10, nu_2=0), True, True),
    "v1_n1": (dict(_V1, n=1, instances=3), True, True),
    "v1_n4": (dict(_V1, n=4), True, True),
    # version 1 with t_exp_left != t_exp_right: right-hand expansion keys on the version-1 path
    "v1_lr": (dict(_V1, t_exp_right=8), True, True),
    # digits past bit 64 (k * bits >= 64): t = 14 (5-bit digits) and 28 (3-bit digits)
    "t14": (dict(t_gsw=14, t_conv=14, t_exp_left=14, t_exp_right=28), True, True),
    "t_mixed": (dict(t_gsw=11, t_conv=13, t_exp_left=20, t_exp_right=29), True, True),
    # 1-bit digits: 112 products per fold accumulator
    "tgsw56": (dict(t_gsw=56, nu_2=1), True, True),
    "p16_q14": (dict(p=16, q2_bits=14), True, True),
    "p2_q16": (dict(p=2, q2_bits=16), True, True),
    # first dimension shorter than one 32-wide k-tile
    "nu1_1": (dict(nu_1=1), True, True),
    "nu1_2": (dict(nu_1=2, nu_2=4), True, True),
    "nu1_4": (dict(nu_1=4), True, True),
    # spiral-rs util.rs no-expansion test parameters with n = 4 (direct upload)
    "direct_n4": (dict(n=4, p=1 << 16, q2_bits=27, t_gsw=3, t_conv=56, t_exp_left=56, t_exp_right=56, nu_2=3), False, True),
    # noise-limited: bytes only
    "t4": (dict(t_gsw=4, t_conv=4, t_exp_left=4, t_exp_right=4), True, False),
    "tgsw3": (dict(t_gsw=3), True, False),
    "p65536_q27": (dict(p=1 << 16, q2_bits=27), True, False),
    "p2_20_q36": (dict(p=1 << 20, q2_bits=36), True, False),
}


def kw(name):
    over, _, _ = SETS[name]
    d = dict(BASE)
    d.update(over)
    return d


def expand(name):
    return SETS[name][1]


def decodes(name):
    return SETS[name][2]
