"""The host side of TrainItemEmbedding (ctr_item_emb_train): ItemSeqGenerator's messages as one int64 stream."""
import numpy as np
import pytest

import go_ctr_b200 as g
from tests.util import INT64_MAX, INT64_MIN


def test_ints_and_canonical_decimal_strings_are_one_stream():
    seq = [7, "7", np.int64(-3), "-3", str(INT64_MIN), INT64_MAX, "0", np.int32(12)]
    got = g.item_ids_from_seq(seq)
    assert got.dtype == np.int64
    assert got.tolist() == [7, 7, -3, -3, INT64_MIN, INT64_MAX, 0, 12]


@pytest.mark.parametrize("bad", ["007", "+7", " 7", "7 ", "-0", "1_000", "7.0", "", "x", str(INT64_MAX + 1), INT64_MIN - 1,
                                 7.0, True, None])
def test_words_that_are_not_a_canonical_int64_are_refused(bad):
    """"007" is a different word from "7" in the reference's string-keyed dictionary: merging them would be silent."""
    with pytest.raises(ValueError):
        g.item_ids_from_seq(["7", bad])


def test_the_entry_point_is_exported():
    assert "ctr_item_emb_train" in g.EXPORTS
    assert g.load_library().ctr_item_emb_train is not None
