"""The streaming kernel's cluster launch: clusters of 8 CTAs, kv head h on cluster h, and the split-KV partials of a kv head
handed to its split 0 through distributed shared memory instead of L2 exchange words.  Only the route of a value changes, so
the committed fixture (tests/golden/stream_digests.json) must hold bit for bit on the cluster path at every legal width, a
Nano-168M decode must equal the plain launch's, widths the cluster launch cannot run are refused, and shapes it does not
take keep the plain launch."""
import re
import subprocess

import numpy as np
import pytest

import bench
from nano_b200 import build as nb_build
from nano_b200 import engine as E, modelfile as mf
from tools import stream_golden as sg

C = 8                  # kStCluster (stream_args.h)
EINVAL = -1            # NB200_EINVAL (include/nano_b200.h)


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _engine(path, S, monkeypatch, **env):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, str(v))
        return E.Engine(path, S)


def _fixture():
    import json
    with open(sg.FIXTURE) as f:
        return json.load(f)


def _widest(path, S, monkeypatch):
    """The cluster launch's widest legal width, found without timing anything: forced widths (no calibration) from the
    largest multiple of 8 on the GPU downward, with the cluster launch required, until the engine accepts one.  How many
    clusters of 8 are resident at once differs between H100s (how their SMs fall into GPCs)."""
    for w in range(_num_sms() // C * C, 0, -C):
        try:
            eng = _engine(path, S, monkeypatch, NB200_STREAM="1", NB200_STREAM_CLUSTER=C, NB200_STREAM_WIDTH=w)
        except E.NB200Error as ex:
            assert f"nb200 error {EINVAL}:" in str(ex) and "NB200_STREAM_CLUSTER" in str(ex), str(ex)
            continue
        try:
            return eng.stream_width, eng.stream_cluster
        finally:
            eng.close()
    raise AssertionError("no width runs the cluster launch")


@pytest.mark.gpu
@pytest.mark.parametrize("case", sg.CASES, ids=[c[0] for c in sg.CASES])
def test_fixture_on_the_cluster_path(case, monkeypatch):
    """Every fixture case at the narrowest (KV clusters) and the widest legal cluster width equals the plain launch's digests."""
    cid, preset, quant, gs, extra, S = case
    spec = mf.PRESETS[preset]
    path = mf.cached_model(spec, quant, gs)
    wmax, cl = _widest(path, S, monkeypatch)
    assert cl == C and wmax % C == 0 and wmax <= _num_sms(), (wmax, cl)
    want = _fixture()[cid]
    for w in sorted({spec.n_kv_head * C, wmax}):
        env = {**extra, "NB200_STREAM_CLUSTER": str(C), "NB200_STREAM_WIDTH": str(w)}
        eng = _engine(path, S, monkeypatch, NB200_STREAM="1", **env)
        assert (eng.stream_width, eng.stream_cluster) == (w, C), (eng.stream_width, eng.stream_cluster)
        eng.close()
        got = sg.run_case((cid, preset, quant, gs, env, S))
        assert got["path"].startswith("streaming"), got["path"]
        bad = [p for p, (a, b) in enumerate(zip(got["logits"], want["logits"])) if a != b]
        assert not bad, f"{cid} at {w} CTAs in clusters: logits differ from the fixture at positions {bad[:8]} ({len(bad)} in all)"
        bad_kv = sorted(k for k in want["kv"] if got["kv"].get(k) != want["kv"][k])
        assert not bad_kv, f"{cid} at {w} CTAs in clusters: K / V rows differ from the fixture at layer/pos {bad_kv}"


def _nano_run(eng, wl):
    preset, _q, _gs, seq = bench.WORKLOADS[wl]
    ids = bench.prompt_ids(mf.PRESETS[preset], seq)
    eng.decode_greedy(ids, bench.PROMPT, seq)
    spec = mf.PRESETS[preset]
    kv = [(eng.read(E.F_KROW, spec.kv_dim, l, p), eng.read(E.F_VROW, spec.kv_dim, l, p))
          for l in (0, spec.n_layer - 1) for p in (0, seq // 2, seq - 2)]
    return ids, eng.logits(), kv


@pytest.mark.gpu
def test_nano168m_cluster_path_equals_plain_launch(monkeypatch):
    """bench.py's headline run: the default engine runs the cluster launch and reports it; at every legal cluster width the
    ids, last logits and K/V rows equal, bit for bit, those of the plain launch (NB200_STREAM_CLUSTER=0)."""
    wl = "nano-168m-q80"
    preset, _q, _gs, seq = bench.WORKLOADS[wl]
    path = bench.model_path(wl)
    KV = mf.PRESETS[preset].n_kv_head
    cal = E.Engine(path, seq)
    assert cal.stream_cluster == C and cal.stream_width % C == 0, (cal.stream_width, cal.stream_cluster)
    print(f"calibrated: {cal.stream_width} CTAs in clusters of {cal.stream_cluster}")
    cal.close()
    plain = _engine(path, seq, monkeypatch, NB200_STREAM_CLUSTER=0, NB200_STREAM_WIDTH=120)
    assert (plain.stream_width, plain.stream_cluster) == (120, None)
    ref = _nano_run(plain, wl)
    plain.close()
    wmax, _ = _widest(path, seq, monkeypatch)
    # the resident clusters of 8 differ between H100s: 14 or 15 on the cards measured
    widths = sorted({w for w in (KV * C, 96, 112, 120, 128) if w <= wmax} | {wmax})
    assert wmax >= 112, widths
    for w in widths:
        eng = _engine(path, seq, monkeypatch, NB200_STREAM_CLUSTER=C, NB200_STREAM_WIDTH=w)
        assert (eng.stream_width, eng.stream_cluster) == (w, C)
        got = _nano_run(eng, wl)
        eng.close()
        assert np.array_equal(got[0], ref[0]), f"ids differ at {w} CTAs"
        assert np.array_equal(got[1].view(np.uint32), ref[1].view(np.uint32)), f"logits differ at {w} CTAs"
        for (ka, va), (kb, vb) in zip(got[2], ref[2]):
            assert np.array_equal(ka.view(np.uint32), kb.view(np.uint32)) and np.array_equal(va.view(np.uint32), vb.view(np.uint32)), w


@pytest.mark.gpu
def test_widths_the_cluster_launch_cannot_run_are_refused(monkeypatch):
    """With the cluster launch required: a width that is not a multiple of 8, fewer CTAs than KV clusters, or more clusters
    than are resident at once is NB200_EINVAL at creation.  Without the requirement such a width runs the plain launch."""
    path = mf.cached_model(mf.PRESETS["long-nano"], mf.QUANT_Q80, 128)          # 8 kv heads; 96 positions: 2 splits
    wmax, _ = _widest(path, 96, monkeypatch)
    bad = [100, 8 * C - C] + ([wmax + C] if wmax + C <= _num_sms() else [])
    for w in bad:
        with pytest.raises(E.NB200Error) as ex:
            _engine(path, 96, monkeypatch, NB200_STREAM_CLUSTER=C, NB200_STREAM_WIDTH=w)
        assert f"nb200 error {EINVAL}:" in str(ex.value) and "NB200_STREAM_CLUSTER" in str(ex.value), str(ex.value)
        eng = _engine(path, 96, monkeypatch, NB200_STREAM_WIDTH=w)
        assert (eng.stream_width, eng.stream_cluster) == (w, None)
        eng.close()
    with pytest.raises(E.NB200Error, match="NB200_STREAM_CLUSTER"):
        _engine(path, 96, monkeypatch, NB200_STREAM_CLUSTER=4)


@pytest.mark.gpu
def test_shapes_the_cluster_launch_does_not_take_keep_the_plain_launch(monkeypatch):
    """More than 8 splits per kv head at max_seq (long-nano and long-qwen3 at 2048: 16) or NB200_STREAM_CLUSTER=0: the plain
    launch, unchanged; requiring the cluster launch there is NB200_EINVAL."""
    for preset, quant in (("long-nano", mf.QUANT_Q80), ("long-qwen3", mf.QUANT_Q4K)):
        path = mf.cached_model(mf.PRESETS[preset], quant, 128)
        eng = _engine(path, 2048, monkeypatch, NB200_STREAM="1")
        assert eng.path.startswith("streaming") and eng.stream_cluster is None, (eng.path, eng.stream_cluster)
        eng.close()
        with pytest.raises(E.NB200Error, match="NB200_STREAM_CLUSTER"):
            _engine(path, 2048, monkeypatch, NB200_STREAM="1", NB200_STREAM_CLUSTER=C)
    path = mf.cached_model(mf.PRESETS["long-nano"], mf.QUANT_Q80, 128)
    eng = _engine(path, 96, monkeypatch, NB200_STREAM_CLUSTER=0)
    assert eng.path.startswith("streaming") and eng.stream_cluster is None
    eng.close()


# ---------------------------------------------------------------- CPU: the cluster instantiations keep the register budget
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def _inst(name):
    m = re.search(r"k_decode_streamILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E", name)
    return tuple(int(x) for x in m.groups()) if m else None


# the plain launch's allowances (Q80 with 64-element groups spills two words around the prologue's poll loop)
ALLOWED_STACK = {(0x80, 4, 2): 8, (0x80, 4, 4): 8}
ALLOWED_LOCAL_OPS = {(0x80, 4, 2): 4, (0x80, 4, 4): 4}


def test_stream_instantiations_have_no_stack_frame_and_no_local_memory():
    """All 24 k_decode_stream<QUANT, LPG, KVM, CL> instantiations, told apart by CL (0: plain launch, 8: cluster launch):
    the plain ones stay within their allowances (no stack and no LDL / STL, except Q80 with 64-element groups), the
    cluster ones use no more than their plain counterparts and none at all outside those allowances."""
    res = subprocess.run([CUOBJDUMP, "-res-usage", nb_build.ENGINE_SO], capture_output=True, text=True, check=True).stdout
    stack, lines = {}, res.splitlines()
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m and _inst(m.group(1)):
            stack[_inst(m.group(1))] = int(re.search(r"STACK:(\d+)", lines[i + 1]).group(1))
    sass = subprocess.run([CUOBJDUMP, "-sass", nb_build.ENGINE_SO], capture_output=True, text=True, check=True).stdout
    local, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = _inst(m.group(1))
            if cur:
                local[cur] = 0
            continue
        if cur and re.search(r"\b(LDL|STL)\b", line):
            local[cur] += 1
    cl = sorted(k for k in stack if k[3] == C)
    assert len(cl) == 12 and len([k for k in stack if k[3] == 0]) == 12, sorted(stack)
    for k in sorted(k for k in stack if k[3] == 0):
        assert stack[k] <= ALLOWED_STACK.get(k[:3], 0) and local[k] <= ALLOWED_LOCAL_OPS.get(k[:3], 0), (k, stack[k], local[k])
    for k in cl:
        plain = k[:3] + (0,)
        assert stack[k] <= stack[plain] and local[k] <= local[plain], (k, stack[k], stack[plain], local[k], local[plain])
        if k[:2] != (0x80, 4):
            assert stack[k] == 0 and local[k] == 0, (k, stack[k], local[k])
