"""The row-sharded kernel probe (tests/cuda/shard_probe.cu) without a GPU: it compiles for sm_90a from the engine's
headers, and the PEER attention, k_shard_adam and k_hot_adam instantiations keep their registers (ptxas -v); and the
numpy references of tests/test_gpu_shard_probe.py (tests/shard_ref.py) are checked on small inputs."""
import math
import re
import subprocess

import numpy as np
import pytest

from tests import shard_probe, shard_ref as ref

PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                   r"\s+ptxas info\s+: Used (\d+) registers")


@pytest.fixture(scope="module")
def ptxas():
    so, log = shard_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    return {n.split("(")[0].replace("void ", ""): v for n, v in zip(names, found.values())}


def test_probe_includes_the_engine_headers_and_never_the_comm_layer():
    src = open(shard_probe.SRC).read()
    assert re.findall(r'#include "([^"]+)"', src) == ["attn.cuh", "knn.cuh", "rec.cuh"]
    for word in ("comm_impl", "k_peer_barrier", "ld.acquire", "__nanosleep", "globaltimer"):
        assert word not in src, word


def test_peer_kernels_compile_without_spills(ptxas):
    """A compile, not a run.  Every PEER attention instantiation the engine launches, k_shard_adam and k_hot_adam: no
    stack frame and no spill — except the D = 128 forward (8 lanes x 4 float4), which holds more than the 64 registers
    its launch bounds allow (the engine compiles the same template from the same header with the same flags); its spill
    is bounded here so that it cannot grow unnoticed."""
    want = []
    for m in (0, 1, 2):
        for D in (16, 32, 64, 128):
            f, b, u = shard_probe.lanes(0, 1, D), shard_probe.lanes(1, 1, D), shard_probe.lanes(0, 0, D)
            want.append(("ctr::k_attn_fwd_idx<%d, %d, %d, true>" % (f + (m,)), D))
            want.append(("ctr::k_attn_bwd_idx<%d, %d, %d, true, true>" % (b + (m,)), D))
            # k_attn_fwd_user takes the non-PEER forward map for both instantiations (engine.cu with_user_kernel)
            want.append(("ctr::k_attn_fwd_user<%d, %d, %d, true>" % (u + (m,)), D))
    for name, D in want:
        assert name in ptxas, (name, sorted(k for k in ptxas if "attn" in k))
        stack, st, ld, regs = ptxas[name]
        print("%s: %d registers, %d bytes stack, %d / %d bytes spilled" % (name, regs, stack, st, ld))
        if D == 128 and "fwd_idx" in name:
            assert stack <= 64 and st <= 64 and ld <= 64, (name, ptxas[name])
        else:
            assert (stack, st, ld) == (0, 0, 0), (name, ptxas[name])
    for name in ("ctr::k_shard_adam", "ctr::k_hot_adam", "ctr::k_hot_apply", "ctr::k_apply_table_grad", "ctr::k_hot_pull",
                 "ctr::k_hot_writeback", "ctr::k_hot_own", "ctr::k_gather_rows_f64"):
        assert ptxas[name][:3] == (0, 0, 0), (name, ptxas[name])


def test_summation_bound_holds_for_float32_orders_and_rejects_an_error():
    rng = np.random.default_rng(0)
    for n in (1, 2, 3, 17, 200):
        for _ in range(20):
            t = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(np.float32)
            exact = math.fsum(t.astype(np.float64))
            abs_sum = np.abs(t.astype(np.float64)).sum()
            for order in (np.arange(n), rng.permutation(n), np.argsort(np.abs(t))):
                acc = np.float32(0)
                for x in t[order]:
                    acc = np.float32(acc + x)
                assert ref.within_sum_bound(acc, exact, n, abs_sum)
            if n > 1:          # an error of a percent of the terms' magnitude is far outside the bound
                assert not ref.within_sum_bound(exact + 0.01 * abs_sum, exact, n, abs_sum)
    assert ref.sum_bound(1, 5.0) == 0.0             # one term: the red.add onto a zero row is exact


def test_row_adam64_matches_a_float32_evaluation():
    rng = np.random.default_rng(1)
    n = 1000
    w = rng.standard_normal(n).astype(np.float32); m = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    v = (rng.random(n) * 1e-5).astype(np.float32); g = rng.standard_normal(n).astype(np.float32); g[:10] = 0
    c = dict(lr=np.float32(0.01), b1=np.float32(0.9), b2=np.float32(0.999), eps=np.float32(1e-8),
             c1=np.float32(1 - np.float64(np.float32(0.9)) ** 2), c2=np.float32(1 - np.float64(np.float32(0.999)) ** 2),
             inv_batch=np.float32(1 / 256))
    gs = g * c["inv_batch"]                                # row_adam_elem, step by step in float32
    m32 = c["b1"] * m + (np.float32(1) - c["b1"]) * gs
    v32 = c["b2"] * v + (np.float32(1) - c["b2"]) * gs * gs
    w32 = w - c["lr"] * (m32 / c["c1"]) / (np.sqrt(v32 / c["c2"]) + c["eps"])
    _, m64, v64, tm, tv = ref.row_adam64(w, m, v, g, **c)
    assert (np.abs(m32 - m64) <= tm).all() and (np.abs(v32 - v64) <= tv).all()
    w64, tw = ref.adam_weight_from(w, m32, v32, c["lr"], c["eps"], c["c1"], c["c2"])
    assert (np.abs(w32 - w64) <= tw).all()
    assert (w32[:10] != w[:10]).all()                      # a zero gradient still moves the weight through m
    assert not (np.abs(w32 + 1e-4 - w64) <= tw).all()      # a shifted weight is outside the bar


def test_topk_order():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    s = np.array([0.5, nan, 0.5, 2.0, -inf, 0.5, -1.0, 0.0], np.float32)
    rows = np.array([9, 1, 4, 7, 3, 2, 8, 5], np.int32)
    r, v, n = ref.topk(s, rows, 6, lambda x: x == x)        # recommendation: any logit but NaN
    assert n == 6 and r.tolist() == [7, 2, 4, 9, 5, 8] and v.tolist() == [2.0, 0.5, 0.5, 0.5, 0.0, -1.0]
    r, v, n = ref.topk(s, rows, 8, lambda x: x == x)
    assert n == 7 and r.tolist() == [7, 2, 4, 9, 5, 8, 3, -1] and v[6] == -inf and v[7] == 0
    r, v, n = ref.topk(s, rows, 5, lambda x: x > 0)         # search: similarities > 0 only
    assert n == 4 and r.tolist() == [7, 2, 4, 9, -1]
