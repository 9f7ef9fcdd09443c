"""The streaming kernel's grid width (NB200_STREAM_WIDTH, or the width the engine times fastest at creation) moves rows and
attention items between CTAs but must not change a bit: the committed fixture of tests/golden/stream_digests.json holds at
narrower grids, Nano-168M Q80 decodes bench.py's run identically at the calibrated width and at num_sms, and widths the
kernel cannot run are refused at creation."""
import os
import re

import numpy as np
import pytest

import bench
from nano_b200 import engine as E, modelfile as mf
from tools import stream_golden as sg

pytestmark = pytest.mark.gpu


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fixture():
    import json
    with open(sg.FIXTURE) as f:
        return json.load(f)


def _engine(path, S, monkeypatch, **env):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, str(v))
        return E.Engine(path, S)


def _width_range(path, S, monkeypatch):
    with pytest.raises(E.NB200Error) as ex:
        _engine(path, S, monkeypatch, NB200_STREAM="1", NB200_STREAM_WIDTH=0)
    m = re.search(r"runs on (\d+)\.\.(\d+) CTAs", str(ex.value))
    assert m, str(ex.value)
    return int(m.group(1)), int(m.group(2))


@pytest.mark.parametrize("case", sg.CASES, ids=[c[0] for c in sg.CASES])
def test_fixture_at_narrower_grids(case, monkeypatch):
    """Every fixture case at half of num_sms and at the narrowest width the case allows."""
    cid, preset, quant, gs, extra, S = case
    wmin, wmax = _width_range(mf.cached_model(mf.PRESETS[preset], quant, gs), S, monkeypatch)
    ns = _num_sms()
    assert wmax == ns and wmin < ns // 2, (wmin, wmax)
    want = _fixture()[cid]
    for w in (ns // 2, wmin):
        got = sg.run_case((cid, preset, quant, gs, {**extra, "NB200_STREAM_WIDTH": str(w)}, S))
        assert got["path"].startswith("streaming"), got["path"]
        bad = [p for p, (a, b) in enumerate(zip(got["logits"], want["logits"])) if a != b]
        assert not bad, f"{cid} at {w} CTAs: logits differ from the fixture at positions {bad[:8]} ({len(bad)} in all)"
        bad_kv = sorted(k for k in want["kv"] if got["kv"].get(k) != want["kv"][k])
        assert not bad_kv, f"{cid} at {w} CTAs: K / V rows differ from the fixture at layer/pos {bad_kv}"


def test_nano168m_calibrated_width_decodes_like_full_width(monkeypatch):
    """bench.py's headline run: ids and last logits at the width the engine picked equal those at num_sms, bit for bit."""
    wl = "nano-168m-q80"
    preset, _q, _gs, seq = bench.WORKLOADS[wl]
    spec, path = mf.PRESETS[preset], bench.model_path(wl)
    ns = _num_sms()
    cal = E.Engine(path, seq)
    full = _engine(path, seq, monkeypatch, NB200_STREAM_WIDTH=ns)
    assert full.stream_width == ns and cal.stream_width is not None, (full.stream_width, cal.stream_width)
    print(f"calibrated width {cal.stream_width} of {ns}")
    out = []
    for eng in (cal, full):
        ids = bench.prompt_ids(spec, seq)
        eng.decode_greedy(ids, bench.PROMPT, seq)
        out.append((ids, eng.logits()))
        eng.close()
    assert np.array_equal(out[0][0], out[1][0])
    assert np.array_equal(out[0][1].view(np.uint32), out[1][1].view(np.uint32))


def test_widths_the_kernel_cannot_run_are_refused(monkeypatch):
    """Below KV x splits at the longest range, below n_embd / kStOwnMax or above num_sms: NB200_EINVAL at creation."""
    ns = _num_sms()
    # long-nano at 2048 positions: 8 kv heads x 16 splits = 128 CTAs; at 96 positions 8 x 2 = 16
    path = mf.cached_model(mf.PRESETS["long-nano"], mf.QUANT_Q80, 128)
    assert _width_range(path, 2048, monkeypatch) == (8 * min(16, ns // 8), ns)
    assert _width_range(path, 96, monkeypatch) == (16, ns)
    # n_embd 2560 (Qwen3-4B layers) at 32 positions: at most 128 residual rows per CTA -> 20 CTAs, above 8 kv heads x 1 split
    path4 = mf.cached_model(mf.PRESETS["qwen3-4b-2l"], mf.QUANT_Q80, 128, fast=True)
    assert _width_range(path4, 32, monkeypatch) == (20, ns)
    for w in (15, ns + 1):
        with pytest.raises(E.NB200Error, match="NB200_STREAM_WIDTH"):
            _engine(path, 96, monkeypatch, NB200_STREAM="1", NB200_STREAM_WIDTH=w)
    eng = _engine(path, 96, monkeypatch, NB200_STREAM_WIDTH=16)         # the narrowest runs
    assert eng.stream_width == 16
    ids = np.zeros(97, np.uint32); ids[:4] = [1, 2, 3, 4]
    eng.decode_greedy(ids, 4, 96)
    eng.close()


def test_multikernel_engines_report_no_width(monkeypatch):
    path = mf.cached_model(mf.PRESETS["toy-nano"], mf.QUANT_Q80, 64)
    eng = E.Engine(path, 64, flags=E.FLAG_NO_STREAM)
    assert eng.stream_width is None and not eng.path.startswith("streaming")
    eng.close()
