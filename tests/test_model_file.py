"""CPU suite for the self-contained model file: DD3DB200.save_model_file read back by an independent Python parser of the
layout include/dd3d_b200.h documents (desc bytes, the dd3d_set_* values and every tensor, bit for bit), and
dd3d_create_from_file refusing every kind of defective file with DD3D_ERR_INVALID before any CUDA call."""
import ctypes as C
import hashlib
import os
import re
import struct

import numpy as np
import pytest
import torch

from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle import fpn_inputs_oracle, num_classes_oracle

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_ERR_INVALID, DD3D_ERR_CUDA = -1, -3
HEADER = struct.Struct("<8sIIIIQ")

SAVE_CASES = {
    "dla34_kitti": lambda: get_cfg("dla34", "kitti_3d"),
    "v2_99_nusc": lambda: get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D"),
    "dla34_c26": lambda: num_classes_oracle.case_cfg("dla34_c26"),
    "dla34_fpn_l2_l5_heads_p2_p6": lambda: fpn_inputs_oracle.case_cfg("dla34_l2_l5"),
}


def _model(cfg):
    return (NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200)(cfg)


def _parse(blob):
    """The model file layout of include/dd3d_b200.h, restated."""
    magic, version, desc_bytes, layout_bytes, num_tensors, size = HEADER.unpack_from(blob, 0)
    assert (magic, version, size) == (b"DD3DB200", 1, len(blob))
    assert (desc_bytes, layout_bytes) == (C.sizeof(lib.ModelDesc), C.sizeof(lib.LayoutDesc))
    assert hashlib.blake2b(blob[:-8], digest_size=8).digest() == blob[-8:]
    o = HEADER.size
    out = dict(desc=blob[o:o + desc_bytes], layout=blob[o + desc_bytes:o + desc_bytes + layout_bytes])
    o += desc_bytes + layout_bytes
    out["backbone_norm"], out["fpn_channels"] = struct.unpack_from("<ii", blob, o)
    o += 8
    for key in ("fpn_inputs", "in_features"):
        n, = struct.unpack_from("<I", blob, o)
        out[key] = list(struct.unpack_from(f"<{n}i", blob, o + 4))
        o += 4 + 4 * n
    n, = struct.unpack_from("<I", blob, o)
    out["canonical_sizes"] = np.frombuffer(blob, "<f4", 3 * n, o + 4)
    o += 4 + 12 * n
    out["tensors"] = {}
    for _ in range(num_tensors):
        k, = struct.unpack_from("<I", blob, o)
        name = blob[o + 4:o + 4 + k].decode()
        ndim, = struct.unpack_from("<I", blob, o + 4 + k)
        shape = struct.unpack_from(f"<{ndim}q", blob, o + 8 + k)
        o += 8 + k + 8 * ndim
        count = int(np.prod(shape, dtype=np.int64))
        assert name not in out["tensors"]
        out["tensors"][name] = np.frombuffer(blob, "<f4", count, o).reshape(shape)
        o += 4 * count
    assert o == len(blob) - 8
    return out


@pytest.mark.parametrize("case", list(SAVE_CASES))
def test_save_model_file_reads_back_bit_for_bit(case, tmp_path):
    cfg = SAVE_CASES[case]()
    model = _model(cfg)
    sd = make_state_dict(cfg)
    model.load_state_dict(sd)
    path = tmp_path / "model.dd3d"
    model.save_model_file(str(path))
    got = _parse(path.read_bytes())

    desc = lib.desc_from_cfg(cfg)
    desc.pixel_mean[:] = [float(v) for v in sd["pixel_mean"].reshape(-1)]
    desc.pixel_std[:] = [float(v) for v in sd["pixel_std"].reshape(-1)]
    assert got["desc"] == bytes(desc)
    assert got["layout"] == bytes(lib.layout_from_cfg(cfg))
    assert got["backbone_norm"] == lib.BACKBONE_NORMS[cfg.FE.BACKBONE.NORM]
    assert got["fpn_channels"] == cfg.FE.FPN.OUT_CHANNELS
    for key, from_cfg in (("fpn_inputs", lib.fpn_inputs_from_cfg), ("in_features", lib.in_features_from_cfg)):
        arg = from_cfg(cfg)
        assert got[key] == ([] if arg is None else list(arg[0]))
    if cfg.DD3D.NUM_CLASSES > lib.MAX_CLASSES:
        assert got["canonical_sizes"].tobytes() == bytes(lib.canonical_sizes_from_cfg(cfg))
    else:
        assert got["canonical_sizes"].size == 0
    # every floating-point tensor of the state_dict, in the order load_state_dict keeps, as fp32 bits
    expected = {k: v for k, v in model.state_dict().items() if v.is_floating_point()}
    assert list(got["tensors"]) == list(expected)
    for k, v in expected.items():
        assert got["tensors"][k].shape == tuple(v.shape), k
        assert np.array_equal(got["tensors"][k].view(np.int32), v.to(torch.float32).numpy().view(np.int32)), k
    # the cases cover the optional calls they are named for
    assert bool(got["canonical_sizes"].size) == (case == "dla34_c26")
    assert bool(got["fpn_inputs"]) == bool(got["in_features"]) == (case == "dla34_fpn_l2_l5_heads_p2_p6")
    assert struct.unpack_from("<i", got["desc"], lib.ModelDesc.nuscenes_heads.offset)[0] == (case == "v2_99_nusc")


def test_save_model_file_stores_do_nms_and_the_forward_capacity(tmp_path):
    """do_nms as the model has it at save time, and the output capacity the forward then uses (every candidate)."""
    cfg = get_cfg("dla34", "kitti_3d")
    model = DD3DB200(cfg)
    model.load_state_dict(make_state_dict(cfg))
    model.do_nms = False
    path = tmp_path / "model.dd3d"
    model.save_model_file(str(path))
    desc = lib.ModelDesc.from_buffer_copy(_parse(path.read_bytes())["desc"])
    assert desc.do_nms == 0 and desc.out_cap == lib.max_candidates(cfg) == 5 * 1000


def test_save_model_file_needs_weights(tmp_path):
    with pytest.raises(RuntimeError, match="load_state_dict"):
        DD3DB200(get_cfg("dla34", "kitti_3d")).save_model_file(str(tmp_path / "model.dd3d"))


# ------------------------------------------------------------------------------------------------ refusals
def _small_file(path, tensors=None):
    """A small well-formed file: the DLA-34 desc and layout, every optional list, and three tiny records."""
    cfg = get_cfg("dla34", "kitti_3d")
    if tensors is None:
        tensors = [("a.weight", torch.arange(6, dtype=torch.float32).reshape(2, 3)), ("s", torch.tensor(2.5)),
                   ("b.bias", torch.ones(4))]
    spec = lib.EngineSpec(lib.desc_from_cfg(cfg), lib.layout_from_cfg(cfg), lib.NORM_BN_SHARED, 256,
                          ((C.c_int32 * 3)(3, 4, 5), 3), ((C.c_int32 * 2)(0, 1), 2), (1, (C.c_float * 3)(1.0, 2.0, 3.0)),
                          lambda: tensors)
    lib.write_model_file(str(path), spec)
    return bytearray(path.read_bytes())


def _create(path):
    L = lib.load()
    h = C.c_void_p(1)
    st = L.dd3d_create_from_file(str(path).encode(), C.byref(h))
    msg = (L.dd3d_last_error(None) or b"").decode()
    assert h.value is None  # no handle on any error path
    return st, msg


def _refused(path, blob, pattern):
    path.write_bytes(bytes(blob))
    st, msg = _create(path)
    assert st == DD3D_ERR_INVALID and re.search(pattern, msg), (st, msg)


def _reseal(blob):
    blob[-8:] = hashlib.blake2b(bytes(blob[:-8]), digest_size=8).digest()
    return blob


def _record_offset(blob, name):
    """Offset of the ndim word of the record named `name`."""
    key = struct.pack("<I", len(name)) + name.encode()
    return blob.index(key) + len(key)


def test_small_file_passes_validation_without_gpu(tmp_path):
    """Valid files get past the host checks to dd3d_create, whose error comes back unchanged (DD3D_ERR_CUDA here)."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: tests/test_model_file_gpu.py covers the calls after validation")
    path = tmp_path / "m.dd3d"
    _small_file(path)
    st, msg = _create(path)
    assert st == DD3D_ERR_CUDA and msg.startswith("dd3d_create: "), (st, msg)


def test_every_truncation_is_refused(tmp_path):
    src = _small_file(tmp_path / "m.dd3d")
    bad = tmp_path / "cut.dd3d"
    for n in range(len(src)):
        _refused(bad, src[:n], r"^model file truncated: %d bytes, \d+ expected$" % n)


def test_corrupt_bytes_fail_the_checksum(tmp_path):
    src = _small_file(tmp_path / "m.dd3d")
    bad = tmp_path / "bad.dd3d"
    for i in list(range(len(src) - 8, len(src))) + [HEADER.size + 4, len(src) - 12]:  # the checksum, the desc, a tensor
        blob = bytearray(src)
        blob[i] ^= 0x10
        _refused(bad, blob, "checksum mismatch")


def test_header_defects(tmp_path):
    src = _small_file(tmp_path / "m.dd3d")
    bad = tmp_path / "bad.dd3d"
    _refused(bad, b"DD3DB201" + src[8:], "bad magic")
    _refused(bad, b"not a model file at all, but long enough to hold a header", "bad magic")
    blob = bytearray(src)
    struct.pack_into("<I", blob, 8, 2)
    _refused(bad, blob, r"unknown model file version 2 \(this library reads version 1\)")
    for field in (12, 16):  # dd3d_model_desc / dd3d_layout_desc sizes of another struct layout
        blob = bytearray(src)
        struct.pack_into("<I", blob, field, struct.unpack_from("<I", src, field)[0] + 4)
        _refused(bad, _reseal(blob), "struct size mismatch")
    _refused(bad, src + b"\0", "1 bytes after its checksum")


def test_record_defects(tmp_path):
    src = _small_file(tmp_path / "m.dd3d")
    bad = tmp_path / "bad.dd3d"
    o = _record_offset(src, "b.bias")  # the last record: ndim 1, shape [4], 16 data bytes
    for shape, pattern in (([5], "shape overruns the file"), ([1 << 62], "shape overruns the file"),
                           ([-4], "negative dimension -4")):
        blob = bytearray(src)
        struct.pack_into("<q", blob, o + 4, *shape)
        _refused(bad, _reseal(blob), r"tensor record 2 \('b.bias'\)(: | )" + pattern)
    for ndim, pattern in ((4, "shape overruns the file"), (9, "ndim 9 out of range")):
        blob = bytearray(src)
        struct.pack_into("<I", blob, o, ndim)
        _refused(bad, _reseal(blob), pattern)
    blob = bytearray(src)  # a name length past the end
    struct.pack_into("<I", blob, o - len("b.bias") - 4, 1 << 20)
    _refused(bad, _reseal(blob), r"tensor record 2 name overruns the file")
    blob = bytearray(src)  # one record fewer in the header: bytes left over
    struct.pack_into("<I", blob, 20, 2)
    _refused(bad, _reseal(blob), "bytes after its last tensor record")
    blob = bytearray(src)  # one record more in the header
    struct.pack_into("<I", blob, 20, 4)
    _refused(bad, _reseal(blob), r"tensor record 3 name length overruns the file")
    blob = bytearray(src)  # a list count past the end
    struct.pack_into("<I", blob, HEADER.size + C.sizeof(lib.ModelDesc) + C.sizeof(lib.LayoutDesc) + 8, 1 << 30)
    _refused(bad, _reseal(blob), "FPN input list overruns the file")


def test_duplicate_names_are_refused(tmp_path):
    t = torch.ones(3)
    path = tmp_path / "dup.dd3d"
    _refused(path, _small_file(path, [("x", t), ("y", t), ("x", t)]), r"duplicate tensor name 'x' \(tensor record 2\)")


def test_unreadable_files_are_refused(tmp_path):
    st, msg = _create(tmp_path / "missing.dd3d")
    assert st == DD3D_ERR_INVALID and "cannot open" in msg and "No such file" in msg
    st, msg = _create(tmp_path)
    assert st == DD3D_ERR_INVALID and "not a regular file" in msg
    L = lib.load()
    h = C.c_void_p()
    assert L.dd3d_create_from_file(None, C.byref(h)) == DD3D_ERR_INVALID
    assert L.dd3d_out_cap(None) == DD3D_ERR_INVALID


def test_new_symbols_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    L = lib.load()
    for name in ("dd3d_create_from_file", "dd3d_out_cap"):
        assert re.search(rf"\bint {name}\(", hdr) and name in lib.SIGNATURES and hasattr(L, name)
