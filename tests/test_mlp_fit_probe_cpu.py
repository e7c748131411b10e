"""The key-fed fit's minibatch gather on a row-sharded ITEM_EMB, without a GPU: the probe (tests/cuda/mlp_fit_probe.cu)
compiles k_gather_rows<double, RowsByIdx, PEER> for sm_90a from attn.cuh, and ptxas -v shows no stack frame and no spill
in either form."""
import re
import subprocess

from tests import mlp_fit_probe

PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")


def test_fit_gather_compiles_without_spills():
    _, log = mlp_fit_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.replace("void ", ""): v for n, v in zip(names, found.values())}
    for prefix in ("ctr::k_gather_rows<double, ctr::RowsByIdx, false>(", "ctr::k_gather_rows<double, ctr::RowsByIdx, true>("):
        got = {k: v for k, v in props.items() if k.startswith(prefix)}
        assert len(got) == 1, (prefix, sorted(props))
        for name, v in got.items():
            assert v == (0, 0, 0), (name, v)
