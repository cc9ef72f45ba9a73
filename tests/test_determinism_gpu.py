"""Bit-level determinism of the engine (-m gpu; VERDICT r1 weak #3).

 * poison: every byte a kernel reads is written earlier in the same forward -- planning over a zeroed arena and over an
   arena filled with 0xFF (NaN in bf16 / fp16 / fp32) gives bit-identical op outputs, head maps and detections;
 * processes: two fresh processes (one of them with programmatic dependent launch disabled) produce identical hashes of
   every stage (tools/determinism_probe.py).
compute-sanitizer's initcheck cannot replace the poison test: it does not track global memory written by TMA stores
(cp.async.bulk.tensor), so it reports every read of a conv output as uninitialised."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from dd3d_b200 import lib
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.gen_golden import case_cfg, case_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _run(case, dtype, fill, reuse=1, sparse=0):
    cfg = case_cfg(case, act_dtype=dtype)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    L = lib.load()
    h = model._engine()
    lib.check(L.dd3d_set_option(h, b"workspace_fill", fill), h)
    lib.check(L.dd3d_set_option(h, b"workspace_reuse", reuse), h)
    lib.check(L.dd3d_set_option(h, b"sparse_box3d", sparse), h)  # sparse = 0: the snapshot includes the dense 3-D maps
    out = model(case_inputs(case))
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    snap = {"input": _bits(model.get_tensor("input")).clone()}
    for i in range(L.dd3d_num_ops(h)):
        s = 0
        while True:
            try:
                snap[f"op{i}:{s}"] = _bits(model.get_tensor(f"op{i}:{s}")).clone()
            except RuntimeError:
                break
            s += 1
    for l in range(5):
        for n in ("cls", "box") + (() if sparse else ("b3d", )):
            snap[f"{n}{l}"] = _bits(model.get_tensor(f"{n}{l}")).clone()
    for b, o in enumerate(out):
        inst = o["instances"]
        snap[f"dets{b}"] = _bits(torch.cat([inst.pred_boxes.tensor, inst.scores_3d[:, None], inst.pred_boxes3d.quat,
                                            inst.pred_boxes3d.size], 1))
    return snap


@pytest.mark.parametrize("case,dtype", [("dla34", "bf16"), ("v2_99", "bf16"), ("v2_99", "fp16"), ("dla34_full", "fp16")])
def test_poisoned_workspace_changes_nothing(case, dtype):
    a = _run(case, dtype, 0x00)
    b = _run(case, dtype, 0xFF)
    assert a.keys() == b.keys() and len(a) > 40
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), f"{case} {dtype}: {k} depends on the arena contents"
    assert sum(a[k].shape[0] for k in a if k.startswith("dets")) > 0


@pytest.mark.parametrize("case,dtype", [("dla34", "bf16"), ("v2_99", "bf16")])
def test_workspace_liveness_reuse_changes_nothing_but_the_footprint(case, dtype):
    """Activation buffers with disjoint lifetimes share arena memory (default); with reuse off every op output has its own.
    Persistent tensors (input, FPN outputs, head maps) and the detections must be bit-identical; the arena must shrink."""
    a = _run(case, dtype, 0xFF, reuse=1)
    b = _run(case, dtype, 0xFF, reuse=0)
    keep = [k for k in a if not k.startswith("op")]
    assert len(keep) >= 1 + 15 + 1
    for k in keep:
        assert torch.equal(a[k], b[k]), f"{case}: {k} differs between reuse on / off"
    cfg = case_cfg(case, act_dtype=dtype)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    L = lib.load()
    h = model._engine()
    sizes = {}
    for reuse in (1, 0):
        lib.check(L.dd3d_set_option(h, b"workspace_reuse", reuse), h)
        sizes[reuse] = L.dd3d_workspace_bytes(h, 8, 384, 1280)
    assert 0 < sizes[1] < 0.6 * sizes[0], sizes


@pytest.mark.parametrize("case,dtype", [("dla34", "bf16"), ("v2_99", "bf16"), ("dla34_full", "fp16")])
def test_sparse_box3d_path_is_arena_independent(case, dtype):
    """Sparse box3d predictor (at the final candidates only, csrc/b3d_sparse.cu; forced on here): the box3d tower outputs must
    survive in the liveness-packed arena until the sparse predictor has read them, and nothing may depend on what the
    workspace held: zeroed / poisoned arena and reuse on / off give bit-identical detections."""
    a = _run(case, dtype, 0x00, reuse=1, sparse=1)
    b = _run(case, dtype, 0xFF, reuse=1, sparse=1)
    c = _run(case, dtype, 0xFF, reuse=0, sparse=1)
    dets = [k for k in a if k.startswith("dets")]
    assert dets and sum(a[k].shape[0] for k in dets) > 0
    for k in dets:
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), f"{case}: {k}"


def _probe(env_extra):
    env = dict(os.environ, **env_extra)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "determinism_probe.py"), "--case", "dla34"],
                         capture_output=True, text=True, env=env, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    line = [l for l in res.stdout.splitlines() if l.startswith("PROBE ")][-1]
    return json.loads(line[6:])["runs"]


def test_fresh_processes_agree_with_and_without_pdl():
    a = _probe({})
    b = _probe({"DD3D_NO_PDL": "1"})
    assert a[0] == a[1] == b[0] == b[1]
    assert sum(a[0]["counts"]) > 0 and len(a[0]["ops"]) > 50
