"""ctr_mlp_fit_keys_dist on a single-GPU feature store is ctr_mlp_fit_keys: the same model, n_iter, loss curve and
rows_used bit for bit, for the classifier and the regressor, and the same refusals (no keys is CTR_EINVAL there, as one
GPU refuses n < 1; every key unknown is CTR_ENOTFOUND with the parameters unchanged)."""
import numpy as np
import pytest

import go_ctr_b200 as g
from tests.test_gpu_mlp64_keys import Store, assert_same_fit

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["classifier", "regressor"])
def test_world_one_is_fit_keys(kind):
    rng = np.random.default_rng(21)
    st = Store(rng)
    u, i, t, y = st.keys(rng, 900)
    if kind == "regressor":
        y = rng.integers(1, 6, u.size).astype(np.float32)
    cls = g.MLPClassifier if kind == "classifier" else g.engine.MLPRegressor
    kw = dict(hidden=(12, 5), max_iter=3, seed=2, tol=0.0, batch=64)
    md = cls(st.nin, **kw).fit_keys_dist(st.eng, u, i, t, y)
    mk = cls(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    assert 0 < md.rows_used < u.size
    assert_same_fit(md, mk, mk.rows_used)
    with pytest.raises(g.CtrError) as e:
        md.fit_keys_dist(st.eng, u[:0], i[:0], t[:0], y[:0])
    assert e.value.code == g.EINVAL
    before = md.get_params()
    with pytest.raises(g.CtrError) as e:
        md.fit_keys_dist(st.eng, np.full(5, 10**16), i[:5], t[:5], y[:5])
    assert e.value.code == g.ENOTFOUND
    assert np.array_equal(md.get_params().view(np.uint64), before.view(np.uint64))
