"""TestSubmitChecker (submitcheck_test.go:28-429) through SubmitChecker over the dry-run NodeDb on the GPU."""
import pytest

import submit_checker_cases as sc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(sc.CASES))
def test_submit_checker_gpu(name):
    sc.replay(name)
