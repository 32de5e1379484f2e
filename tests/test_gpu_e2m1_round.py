"""The device build of the branch-free E2M1 rounding equals the reference's compare chain on every non-negative fp32
bit pattern (finite, +inf and NaN)."""

import pytest

pytestmark = pytest.mark.gpu


def test_e2m1_round_selftest():
    from model_optimizer_b200 import ops

    assert ops.selftest_e2m1_round() == 0
