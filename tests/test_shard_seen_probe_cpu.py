"""The CTR_EXCLUDE_SEEN kernels, generalised to a row-sharded ITEM_EMB, without a GPU: the probe
(tests/cuda/shard_seen_probe.cu) compiles them for sm_90a from ubcache.cuh and rec.cuh, and ptxas -v shows no stack
frame and no spill for either form of each, the (world, rank) one and the single-table one."""
import re
import subprocess

from tests import shard_seen_probe

PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")


def test_seen_kernels_compile_without_spills():
    _, log = shard_seen_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.replace("void ", ""): v for n, v in zip(names, found.values())}
    want = {
        "ctr::k_ub_seen(": 1,
        "ctr::rec::k_rec_scan_seen<ctr::knn::LogitKey>(": 2,
        "ctr::rec::k_rec_target_logits<float>(": 1,
        "ctr::rec::k_rec_rank_sort_seen<ctr::knn::LogitKey>(": 2,
        "ctr::rec::k_rec_rank_seen<ctr::knn::LogitKey>(": 2,
    }
    for prefix, n in want.items():
        got = {k: v for k, v in props.items() if k.startswith(prefix)}
        assert len(got) == n, (prefix, sorted(props))
        for name, v in got.items():
            assert v == (0, 0, 0), (name, v)
    # the (world, rank) forms take two ints more than the single-table ones
    for prefix in ("ctr::rec::k_rec_scan_seen<", "ctr::rec::k_rec_rank_seen<"):
        arity = sorted(k.count(",") for k in props if k.startswith(prefix))
        assert arity[1] == arity[0] + 2, (prefix, arity)
