"""armada_nodedb_add_classes under the SIMT emulator (no GPU); the bodies are in nodedb_append_cases.py."""
import pytest

import emu_lib
import nodedb_append_cases as na


@pytest.mark.parametrize("chunk", [None, 1, 3])
@pytest.mark.parametrize("seed", [1, 2])
def test_appended_classes_answer_like_a_db_made_with_them(seed, chunk):
    sizes = na.check_append_parity(seed, emu_lib.load(), chunk)
    # the input forces reallocations: the creation sizes the class arrays exactly and they double when outgrown,
    # so ending past 4x the creation's count takes two or more (the growth itself is not observable from here)
    assert sizes[-1] > 4 * sizes[0]


def test_failed_append_changes_nothing():
    na.check_failed_append_changes_nothing(emu_lib.load())


def test_unresolved_label_changes_nothing():
    na.check_unresolved_label_changes_nothing(emu_lib.load())
