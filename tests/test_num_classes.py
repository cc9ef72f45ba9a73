"""CPU suite for DD3D.NUM_CLASSES up to 128: parameter inventory against the reference at every case of
oracle/num_classes_oracle.py, the oracle against the reference's own forward, the config / desc / sizes round trip, the
refusals and the new C symbols."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import param_specs
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.gen_golden import inventory_digest
from oracle.num_classes_oracle import NUM_CLASSES_CASES, canonical_sizes, case_cfg, case_inputs, num_classes_cfg
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_CASES = [c for c, v in NUM_CLASSES_CASES.items() if v[2] == "DD3D"]


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "num_classes_inventory.json")) as f:
        return json.load(f)


def _mirror(cfg):
    return (NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200)(cfg)


@pytest.mark.parametrize("case", list(NUM_CLASSES_CASES))
def test_param_specs_match_reference_inventory(case):
    shapes = {k: shape for k, (shape, _) in param_specs(case_cfg(case)).items()}
    assert inventory_digest(shapes) == _inventory()[case]


@pytest.mark.parametrize("case", list(NUM_CLASSES_CASES))
def test_model_state_dict_keys_equal_generator_keys(case):
    cfg = case_cfg(case)
    sd = _mirror(cfg).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == _inventory()[case]
    assert set(sd) == set(make_state_dict(cfg))


@pytest.mark.parametrize("case", DD3D_CASES)
def test_oracle_matches_reference_golden(case):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/num_classes_oracle.py --golden), the bounds of
    tests/test_dla_x.py."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_num_classes.npz"))
    cfg = case_cfg(case)
    out = DD3DOracle(cfg, make_state_dict(cfg)).forward(case_inputs(case))
    total = 0
    for b, o in enumerate(out):
        p = f"{case}/"
        assert o["box2d"].shape[0] == g[f"{p}boxes{b}"].shape[0]
        total += o["box2d"].shape[0]
        assert np.array_equal(o["cls"].numpy(), g[f"{p}classes{b}"])
        assert np.array_equal(o["level"].numpy(), g[f"{p}levels{b}"])
        np.testing.assert_allclose(o["box2d"].numpy(), g[f"{p}boxes{b}"], rtol=1e-4, atol=1e-3)
        np.testing.assert_allclose(o["score"].numpy(), g[f"{p}scores{b}"], rtol=1e-4)
        np.testing.assert_allclose(o["score3d"].numpy(), g[f"{p}scores_3d{b}"], rtol=1e-4)
        if o["box2d"].shape[0]:
            assert quat_dist(o["quat"], g[f"{p}quat{b}"]).max() < 1e-4
        np.testing.assert_allclose(o["tvec"].numpy(), g[f"{p}tvec{b}"], rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(o["size"].numpy(), g[f"{p}size{b}"], rtol=1e-4)
    assert total > 0
    # classes above 16 are predicted: the size rows past the desc's 16 are exercised
    assert int(max(g[f"{case}/classes{b}"].max(initial=0) for b in range(len(out)))) >= 16


def test_golden_detections_reach_high_classes():
    g = np.load(os.path.join(GOLDEN_DIR, "golden_num_classes.npz"))
    cls = np.concatenate([g[k] for k in g.files if k.startswith("v2_19_slim_c128/classes")])
    assert cls.max() >= 64  # the class ids the group BEV NMS used to flag


@pytest.mark.parametrize("n", [1, 5, 16, 17, 26, 64, 128])
def test_desc_and_sizes_round_trip(n):
    cfg = num_classes_cfg("dla34", n)
    d = lib.desc_from_cfg(cfg)
    assert d.num_classes == n
    rows = canonical_sizes(n)
    for c in range(min(n, lib.MAX_CLASSES)):  # the desc keeps its 16 rows
        assert [d.canonical_box3d_sizes[3 * c + k] for k in range(3)] == pytest.approx(rows[c])
    flat = list(lib.canonical_sizes_from_cfg(cfg))
    assert len(flat) == 3 * n
    assert flat == pytest.approx([v for r in rows for v in r])
    m = DD3DB200(cfg)
    assert m.num_classes == n
    assert (m._canon is not None) == (n > lib.MAX_CLASSES)  # at 16 or fewer the desc rows are the engine's sizes


def test_canonical_size_rule_is_distinct_and_positive():
    rows = canonical_sizes(128)
    assert len({tuple(r) for r in rows}) == 128
    assert min(min(r) for r in rows) > 0.5


@pytest.mark.parametrize("n", [129, 200])
def test_too_many_classes_raise_not_implemented(n):
    cfg = num_classes_cfg("dla34", n)
    param_specs(cfg)  # the reference builds it
    with pytest.raises(NotImplementedError, match="128"):
        DD3DB200(cfg)


@pytest.mark.parametrize("n,rows", [(17, 16), (26, 10), (128, 127)])
def test_missing_size_rows_raise_index_error(n, rows):
    cfg = num_classes_cfg("dla34", n)
    cfg.DD3D.FCOS3D.CANONICAL_BOX3D_SIZES = canonical_sizes(rows)
    with pytest.raises(IndexError, match="CANONICAL_BOX3D_SIZES"):
        DD3DB200(cfg)


def test_missing_size_rows_are_fine_without_a_3d_head():
    cfg = num_classes_cfg("dla34", 26)
    cfg.MODEL.BOX3D_ON = False
    cfg.DD3D.FCOS3D.CANONICAL_BOX3D_SIZES = canonical_sizes(3)
    assert DD3DB200(cfg)._canon is None


@pytest.mark.parametrize("n", [0, -1, 129])
def test_create_refuses_class_counts_out_of_range(n):
    """dd3d_create checks num_classes before it touches a device."""
    L = lib.load()
    d = lib.desc_from_cfg(num_classes_cfg("dla34", 5))
    d.num_classes = n
    h = C.c_void_p()
    assert L.dd3d_create(C.byref(d), C.byref(h)) == -1
    assert b"num_classes" in L.dd3d_last_error(None)
    assert not h.value


def test_new_symbols_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"#define DD3D_MAX_NUM_CLASSES 128\b", hdr) and re.search(r"#define DD3D_MAX_CLASSES 16\b", hdr)
    assert re.search(r"int dd3d_set_canonical_sizes\(dd3d_handle h, int32_t num_classes, const float\* h_sizes\);", hdr)
    L = lib.load()
    for name in ("dd3d_set_canonical_sizes", "dd3d_op_b3d_gather", "dd3d_op_b3d_gather_scratch_bytes", "dd3d_op_detect_c",
                 "dd3d_op_detect_c_scratch_bytes"):
        assert name in hdr and name in lib.SIGNATURES and hasattr(L, name)
    assert lib.MAX_NUM_CLASSES == 128 and lib.MAX_CLASSES == 16
    assert len(lib.SIGNATURES["dd3d_op_detect_c"][1]) == len(lib.SIGNATURES["dd3d_op_detect_flags"][1]) + 1
    assert C.sizeof(lib.ModelDesc) == 4 * (2 + 3 + 3 + 12 + 48 + 9)  # the desc keeps its size


def test_scratch_bytes_without_a_device():
    L = lib.load()
    assert L.dd3d_op_detect_c_scratch_bytes(2, 1000, 16) >= L.dd3d_op_detect_scratch_bytes(2, 1000) - 1024
    assert L.dd3d_op_detect_c_scratch_bytes(2, 1000, 128) > L.dd3d_op_detect_c_scratch_bytes(2, 1000, 16)
    assert L.dd3d_op_detect_c_scratch_bytes(2, 1000, 129) == -1
    assert L.dd3d_op_b3d_gather_scratch_bytes(32, 128, 1000) > 0
    assert L.dd3d_op_b3d_gather_scratch_bytes(1, 129, 10) == -1


def test_set_canonical_sizes_without_a_handle_is_refused():
    sizes = (C.c_float * 3)(1.0, 2.0, 3.0)
    assert lib.load().dd3d_set_canonical_sizes(None, 1, sizes) == -1


def test_gathered_kernel_follows_the_static_kernel_rules():
    """csrc/b3d_gather.cu under the checks tests/test_static_kernel_rules.py runs on the other cp.async / mma.sync kernels:
    every kernel starts with the PDL prologue, the prefetch of the next weight block follows a barrier, a second barrier
    retires the readers of a buffer before it is staged again, and the mma.sync fragment code is b3d_sparse.cu's own."""
    csrc = os.path.join(ROOT, "dd3d_b200", "csrc")
    with open(os.path.join(csrc, "b3d_gather.cu")) as f:
        s = f.read()
    kernels = list(re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?([A-Za-z_0-9]+)\s*\(", s))
    assert {m.group(1) for m in kernels} == {"b3d_group_kernel", "b3d_sparse_kernel_gathered"}
    for m in kernels:
        body = s[s.index("{\n", m.end()) + 2:]
        assert body.lstrip().startswith("DD3D_PDL_PROLOGUE();"), m.group(1)
    body = s[s.index("for (", s.index("cp.async.commit_group")):]
    i_sync, i_load = body.index("__syncthreads()"), body.index("stage_slab(")
    assert i_load < i_sync and body[:body.index("asm volatile(\"cp.async.wait_group 0")].count("__syncthreads()") >= 2
    for fn in ("b3d_gather.cu", "b3d_sparse.cu"):
        with open(os.path.join(csrc, fn)) as f:
            src = f.read()
        assert '#include "b3d_mma.cuh"' in src and "b3d_mma::mma_group<FP16>" in src and "b3d_mma::load_a(" in src
        assert "mma.sync.aligned" not in src, f"{fn}: the fragment arithmetic belongs to b3d_mma.cuh"
