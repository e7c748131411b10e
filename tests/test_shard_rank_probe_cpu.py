"""The rank kernels of ctr_rank_items, generalised to a row-sharded ITEM_EMB, without a GPU: the probe
(tests/cuda/shard_rank_probe.cu) compiles them for sm_90a from rec.cuh, and ptxas -v shows no stack frame and no spill."""
import re
import subprocess

from tests import shard_rank_probe

PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                   r"\s+ptxas info\s+: Used (\d+) registers")


def test_rank_kernels_compile_without_spills():
    _, log = shard_rank_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.split("(")[0].replace("void ", ""): v for n, v in zip(names, found.values())}
    for name in ("ctr::rec::k_rec_target_logits<float>", "ctr::rec::k_rec_rank_sort<ctr::knn::LogitKey>",
                 "ctr::rec::k_rec_rank<ctr::knn::LogitKey>", "ctr::rec::k_rec_rank_finish<float>"):
        assert name in props, (name, sorted(k for k in props if "rec" in k))
        assert props[name][:3] == (0, 0, 0), (name, props[name])
