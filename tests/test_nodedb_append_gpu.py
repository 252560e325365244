"""armada_nodedb_add_classes on the GPU; the bodies are in nodedb_append_cases.py."""
import pytest

import nodedb_append_cases as na

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("chunk", [None, 1, 3])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_appended_classes_answer_like_a_db_made_with_them_gpu(seed, chunk):
    na.check_append_parity(seed, None, chunk)


def test_failed_append_changes_nothing_gpu():
    na.check_failed_append_changes_nothing(None)


def test_unresolved_label_changes_nothing_gpu():
    na.check_unresolved_label_changes_nothing(None)
