"""The float64 MLP's serving kernels on a row-sharded ITEM_EMB, without a GPU: the probe (tests/cuda/shard_mlp_probe.cu)
compiles them for sm_90a from attn.cuh, mlp64.cuh and rec.cuh, and ptxas -v shows no stack frame and no spill for any
form: the key-fed gather and the prefix with and without PEER, both layer-0 forms, and the Logit64Key selection and
rank kernels at (world, rank)."""
import re
import subprocess

from tests import shard_mlp_probe

PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")


def test_mlp_shard_kernels_compile_without_spills():
    _, log = shard_mlp_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.replace("void ", ""): v for n, v in zip(names, found.values())}
    want = {
        "ctr::k_gather_rows<double, ctr::RowsAsIs, false>(": 1,
        "ctr::k_gather_rows<double, ctr::RowsAsIs, true>(": 1,
        "ctr::k_mlp64_prefix<false>(": 1,
        "ctr::k_mlp64_prefix<true>(": 1,
        "ctr::k_mlp64_rec_layer0<false>(": 1,
        "ctr::k_mlp64_rec_layer0<true>(": 1,
        "ctr::rec::k_rec_scan<ctr::knn::Logit64Key>(": 1,
        "ctr::rec::k_rec_scan_seen<ctr::knn::Logit64Key>(": 1,
        "ctr::knn::k_knn_merge<ctr::knn::Logit64Key>(": 1,
        "ctr::rec::k_rec_target_logits<double>(": 1,
        "ctr::rec::k_rec_rank_sort<ctr::knn::Logit64Key>(": 1,
        "ctr::rec::k_rec_rank_sort_seen<ctr::knn::Logit64Key>(": 1,
        "ctr::rec::k_rec_rank<ctr::knn::Logit64Key>(": 1,
        "ctr::rec::k_rec_rank_seen<ctr::knn::Logit64Key>(": 1,
        "ctr::rec::k_rec_rank_finish<double>(": 1,
    }
    for prefix, n in want.items():
        got = {k: v for k, v in props.items() if k.startswith(prefix)}
        assert len(got) == n, (prefix, sorted(props))
        for name, v in got.items():
            assert v == (0, 0, 0), (name, v)
    # layer 0 takes the ITEM_FEAT row mapping (fworld, frank) after n_ifeat
    for name in props:
        if name.startswith("ctr::k_mlp64_rec_layer0<"):
            assert "long, int, int, int, int, long, int, double*)" in name, name
