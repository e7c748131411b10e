"""CTR_EXCLUDE_SEEN without a GPU: the exported entry points and modes, the Python-side argument checks, and the new
kernels compiled for sm_90a from rec.cuh / ubcache.cuh with no stack frame and no spill."""
import os
import re
import subprocess

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import shard_probe

NEW = ["ctr_recommend_topk_ex", "ctr_rank_items_ex", "ctr_mlp_recommend_topk_ex", "ctr_mlp_rank_items_ex"]
HEADER = os.path.join(shard_probe.ROOT, "include", "ctr_b200.h")


def test_ex_entry_points_are_declared_and_exported():
    src = open(HEADER).read()
    assert "enum { CTR_EXCLUDE_NONE = 0, CTR_EXCLUDE_WINDOW = 1, CTR_EXCLUDE_SEEN = 2 };" in src
    assert (g.EXCLUDE_NONE, g.EXCLUDE_WINDOW, g.EXCLUDE_SEEN) == (0, 1, 2)
    assert "#define CTR_B200_ABI_VERSION 1" in src
    L = g.load_library()
    for name in NEW:
        assert re.search(r"\b%s\(" % name, src), name
        assert name in g.EXPORTS and hasattr(L, name), name


def test_exclusion_arguments():
    ex = g.engine._exclusion
    assert ex(3, None, False, False) == (g.EXCLUDE_NONE, None)
    assert ex(3, [1, 2, 3], True, False) == (g.EXCLUDE_WINDOW, None)          # max_ts is not read without exclude_seen
    for hist in (False, True):                                                 # exclude_seen implies exclude_history
        mode, t = ex(3, None, hist, True)
        assert mode == g.EXCLUDE_SEEN and t.dtype == np.int64 and t.tolist() == [0, 0, 0]
    mode, t = ex(2, -2 ** 63, True, True)
    assert t.tolist() == [-2 ** 63, -2 ** 63] and t.flags.c_contiguous
    mode, t = ex(3, np.array([9, 2 ** 63 - 1, 0, 5])[:3], True, True)
    assert t.tolist() == [9, 2 ** 63 - 1, 0]
    for bad in ([1, 2], [[1, 2, 3]], np.zeros((3, 1))):
        with pytest.raises(ValueError):
            ex(3, bad, True, True)


PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
KERNELS = '''#include "rec.cuh"
#include "ubcache.cuh"
using namespace ctr;
template __global__ void rec::k_rec_scan_seen<knn::LogitKey>(const float*, int, int, int, const unsigned*, int, const float*, const int*, float*, int*);
template __global__ void rec::k_rec_scan_seen<knn::Logit64Key>(const double*, int, int, int, const unsigned*, int, const double*, const int*, double*, int*);
template __global__ void rec::k_rec_rank_sort_seen<knn::LogitKey>(const int*, const float*, int, long, const unsigned*, int*, int*, float*, int*, unsigned long long*);
template __global__ void rec::k_rec_rank_sort_seen<knn::Logit64Key>(const int*, const double*, int, long, const unsigned*, int*, int*, double*, int*, unsigned long long*);
template __global__ void rec::k_rec_rank_seen<knn::LogitKey>(const float*, int, int, const unsigned*, const float*, const int*, const int*, unsigned long long*);
template __global__ void rec::k_rec_rank_seen<knn::Logit64Key>(const double*, int, int, const unsigned*, const double*, const int*, const int*, unsigned long long*);
'''


def test_seen_kernels_compile_without_spills(tmp_path):
    nvcc = shard_probe._nvcc()
    if nvcc is None:
        pytest.skip("no nvcc")
    src = tmp_path / "seen_kernels.cu"
    src.write_text(KERNELS)
    flags = [f for f in shard_probe._library_flags() if f not in ("-shared", "-ldl")]
    r = subprocess.run([nvcc] + flags + ["-cubin", "-Xptxas", "-v", "-I", shard_probe.CSRC, "-o", str(tmp_path / "k.cubin"), str(src)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(r.stdout)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.split("(")[0].replace("void ", ""): v for n, v in zip(names, found.values())}
    want = ["ctr::k_ub_seen"] + ["ctr::rec::%s<ctr::knn::%s>" % (k, key) for k in ("k_rec_scan_seen", "k_rec_rank_sort_seen", "k_rec_rank_seen")
                                 for key in ("LogitKey", "Logit64Key")]
    for name in want:
        assert name in props, (name, sorted(props))
        assert props[name] == (0, 0, 0), (name, props[name])
