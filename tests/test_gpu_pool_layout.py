"""GPU: what every pool looks like from outside -- its state and action keys, slab size, state
blob layout (the snapshot format), bytes_per_env_step, the launch count after creation, and
the errors of the configurations it rejects -- against tests/golden/pool_layouts.json, for
every kind, both precisions, num_envs 1 and 1000 and every iopt (tests/golden/
make_pool_layouts.py records the fixture and lists the cases)."""
import json
import os
import sys

import pytest

from envpool_b200 import _capi
from helpers import GOLDEN

sys.path.insert(0, GOLDEN)
from make_pool_layouts import FIXTURE, cases, describe  # noqa: E402

CASES = dict(cases(_capi.KINDS))

with open(FIXTURE) as f:
    WANT = json.load(f)


def test_fixture_covers_every_case():
    assert sorted(WANT) == sorted(CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_pool_layout(capi, case):
    assert describe(capi, *CASES[case]) == WANT[case]
