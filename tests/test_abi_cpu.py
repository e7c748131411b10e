"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/ctr_b200.h declares, and refuses to run without an H100 (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import go_ctr_b200 as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "ctr_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ctr_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_loads():
    import __graft_entry__ as ge
    ge.build()
    lib = g.load_library()
    assert lib.ctr_abi_version() == 1


def test_every_declared_symbol_is_exported():
    lib = g.load_library()
    declared = _header_functions()
    assert sorted(g.EXPORTS) == declared, set(g.EXPORTS) ^ set(declared)
    for name in declared:
        assert getattr(lib, name) is not None


def test_config_default_carries_reference_hyperparameters():
    cfg = g.engine.default_config(g.MODEL_DIN_COS)
    assert (cfg.H0, cfg.H1, cfg.S, cfg.D) == (200, 80, 10, 16)              # din.go:17-18, rcmd.go:22-24
    assert abs(cfg.lr - 0.01) < 1e-9 and abs(cfg.l2 - 1e-4) < 1e-9          # model.go:88
    assert abs(cfg.dropout0 - 0.005) < 1e-9                                  # din.go:204
    assert abs(g.engine.default_config(g.MODEL_YOUTUBE).dropout0 - 0.003) < 1e-9   # dnn.go:136


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(g.CtrError) as e:
        g.Engine(g.engine.default_config(g.MODEL_DIN_COS))
    assert e.value.code == 2 and "no CPU fallback" in str(e.value)          # CTR_ENODEV


def test_bad_config_is_an_error_code_not_an_abort():
    lib = g.load_library()
    cfg = g.engine.default_config(g.MODEL_DIN_COS, S=0)
    h = C.c_void_p()
    assert lib.ctr_create(C.byref(cfg), C.byref(h)) == 1                     # CTR_EINVAL
    assert b"bad dims" in lib.ctr_last_error(None)


def test_dim_mismatch_is_the_reference_error():
    with pytest.raises(ValueError, match="uBehaviorDim 7 != iFeatureDim 8"):   # din.go:176-178
        g.NewDinNet(5, 3, 7, 8, 5)


def test_marshal_schema_matches_reference_json():
    import json
    import numpy as np
    net = g.NewDinNet(5, 3, 7, 7, 5)
    inn = 5 + 7 + 7 + 5
    net.weights = (np.arange(inn * 200, dtype=np.float32).reshape(inn, 200), np.ones((200, 80), np.float32),
                   np.ones((80, 1), np.float32), np.array([1, 2, 3], np.float32))
    m = json.loads(net.Marshal())
    assert list(m) == ["uProfileDim", "uBehaviorSize", "uBehaviorDim", "iFeatureDim", "cFeatureDim", "mlp0", "mlp1", "mlp2", "att0"]   # din.go:41-52
    back = g.NewDinNetFromJson(net.Marshal())
    assert back.d0 == 0.0 and back.d1 == 0.0                                 # din.go:133-145
    np.testing.assert_array_equal(back.weights[0], net.weights[0])
    y = g.NewYoutubeDnn(5, 3, 7, 7, 5); y.weights = net.weights
    assert "att0" not in json.loads(y.Marshal())                             # dnn.go:38-47


def test_idmap_hash_restatement_and_its_inverse():
    """tests/util.py restates idmap.cuh's idmap_hash in numpy and inverts it, so that test_gpu_keys.py can build ids
    that start their probe at chosen slots.  Checked here against a plain-integer transcription of the device function."""
    import numpy as np
    from tests.util import INT64_MAX, INT64_MIN, idmap_capacity, idmap_hash, idmap_unhash, ids_probing_from

    M = (1 << 64) - 1

    def fmix64(k):                       # idmap_hash, line for line
        k ^= k >> 33; k = k * 0xff51afd7ed558ccd & M; k ^= k >> 33; k = k * 0xc4ceb9fe1a85ec53 & M; k ^= k >> 33
        return k

    rng = np.random.default_rng(5)
    ids = np.concatenate([[0, -1, 1, INT64_MAX, INT64_MIN, INT64_MIN + 1], rng.integers(INT64_MIN, INT64_MAX, 2000, dtype=np.int64)])
    assert idmap_hash(ids).tolist() == [fmix64(int(v) & M) for v in ids]
    assert (idmap_unhash(idmap_hash(ids)) == ids).all()
    h = np.concatenate([np.array([0, 1, 1 << 63, M], np.uint64), rng.integers(0, 2**64, 2000, dtype=np.uint64)])
    assert (idmap_hash(idmap_unhash(h)) == h).all()
    assert [idmap_capacity(n) for n in (1, 32, 33, 64, 65, 100_000)] == [64, 64, 128, 128, 256, 262_144]
    for cap in (64, 128, 262_144):
        slots = np.concatenate([np.full(20, cap - 1), np.arange(20), rng.integers(0, cap, 20)])
        got = ids_probing_from(rng, slots, cap, avoid=[0, -1])
        assert ((idmap_hash(got) & np.uint64(cap - 1)) == slots.astype(np.uint64)).all()
        assert np.unique(got).size == got.size and not np.isin(got, [INT64_MIN, 0, -1]).any()


def test_item2vec_host_plan_matches_the_reference_huffman_procedure():
    """ctr_i2v_paths (host-only part of the item2vec trainer) == dictionary.HuffnamTree + Node.GetPath as the
    oracle restates them (huffman.go:23-57, node.go:26-43), including ties and never-seen words."""
    import time
    import numpy as np
    from oracle import oracle as orc
    rng = np.random.default_rng(0)
    for V, hi in ((2, 5), (9, 3), (300, 4), (2000, 100000)):
        cnt = rng.integers(0, hi, V); cnt[0] = max(cnt[0], 1)
        off, nodes, codes = g.i2v_paths(cnt)
        parent, code = orc.i2v_huffman(cnt, literal=True)
        for w in range(V):
            n, c = orc.i2v_path(parent, code, V, w)
            if cnt[w] == 0:           # an id that never occurs is not a dictionary word in the reference: in the tree, but no path is built
                assert off[w] == off[w + 1]
                continue
            assert nodes[off[w]:off[w + 1]].tolist() == n.tolist() and codes[off[w]:off[w + 1]].tolist() == c.tolist(), (V, hi, w)
    off, nodes, _ = g.i2v_paths(np.ones(50, np.int64), max_depth=3)
    assert (np.diff(off) == 2).all()                                   # GetPath(3) → two (node, code) steps
    cnt = np.floor(np.exp(rng.random(400000) * np.log(50))).astype(np.int64) - 1   # ~half zeros, heavy ties
    t0 = time.perf_counter(); g.i2v_paths(cnt); assert time.perf_counter() - t0 < 20   # no quadratic insertion
