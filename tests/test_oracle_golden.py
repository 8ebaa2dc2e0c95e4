"""The CPU oracle against every golden vector the reference's own tests hold for
the coverage path.  Runs without a GPU."""
import os

import pytest

from case_runner import ORACLE_BIN, check_case, run_case
from reference_cases import ALL_CASES


@pytest.fixture(scope="session", autouse=True)
def _oracle_built():
    if not os.path.exists(ORACLE_BIN):
        import subprocess
        subprocess.check_call(["make", "-C", os.path.dirname(ORACLE_BIN)])


@pytest.mark.parametrize("case", ALL_CASES, ids=[f"{c['sub']}@{c['ref']}" for c in ALL_CASES])
def test_oracle_matches_reference_golden(case):
    check_case(case, run_case(ORACLE_BIN, case))
