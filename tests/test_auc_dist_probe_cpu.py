"""The per-rank kernels of ctr_roc_auc_dist and ctr_group_auc_dist without a GPU: the probe (tests/cuda/auc_dist_probe.cu)
compiles them for sm_90a from auc.cuh, and ptxas -v shows no stack frame and no spill in any of them."""
import re
import subprocess

from tests import auc_dist_probe

PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
KERNELS = ["ctr::k_auc_dist_keys(", "ctr::k_auc_dist_area(", "ctr::k_gauc_dist_rec(", "ctr::k_dist_samples<unsigned int>(",
           "ctr::k_dist_samples<unsigned long long>(", "ctr::k_dist_part<unsigned int>(", "ctr::k_dist_part<unsigned long long>("]


def test_dist_kernels_compile_without_spills():
    _, log = auc_dist_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.replace("void ", ""): v for n, v in zip(names, found.values())}
    for prefix in KERNELS:
        got = {k: v for k, v in props.items() if k.startswith(prefix)}
        assert len(got) == 1, (prefix, sorted(props))
        for name, v in got.items():
            assert v == (0, 0, 0), (name, v)
