"""The streaming decode kernel against a committed bit-exact fixture (tests/golden/stream_digests.json, recipe in
tools/stream_golden.py): sha256 digests of every position's logits and of K / V rows of every layer, on seeded 2-layer
models that put the O and W2 phases on shared and on warp-owned tiles, with Q80 groups of 64 and 128 and with Q4K.

The O and W2 operands are quantised group by group as their exchange words arrive, and each row dot waits for its own
group; none of that may change a code, a scale or the order of any fp32 sum, so the kernel must reproduce the fixture
bit for bit."""
import json

import pytest

from tools import stream_golden as sg


def _fixture():
    with open(sg.FIXTURE) as f:
        return json.load(f)


def test_fixture_covers_every_case():
    got = _fixture()
    assert sorted(got) == sorted(c[0] for c in sg.CASES)
    for c in sg.CASES:
        assert len(got[c[0]]["logits"]) == c[5]


@pytest.mark.gpu
@pytest.mark.parametrize("case", sg.CASES, ids=[c[0] for c in sg.CASES])
def test_stream_kernel_matches_fixture(case):
    want = _fixture()[case[0]]
    got = sg.run_case(case)
    assert got["path"].startswith("streaming"), f"expected the streaming kernel, engine runs: {got['path']}"
    bad = [p for p, (a, b) in enumerate(zip(got["logits"], want["logits"])) if a != b]
    assert not bad, f"{case[0]}: logits differ from the fixture at positions {bad[:8]} ({len(bad)} in all)"
    bad_kv = sorted(k for k in want["kv"] if got["kv"].get(k) != want["kv"][k])
    assert not bad_kv, f"{case[0]}: K / V rows differ from the fixture at layer/pos {bad_kv}"
