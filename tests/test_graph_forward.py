"""The CUDA-graph forward's C ABI without a device: dd3d_graph_create / dd3d_graph_launch / dd3d_graph_destroy /
dd3d_graph_kernel_nodes / dd3d_graph_programmatic_edges are declared in include/dd3d_b200.h and exported by the library,
and NULL handles and graphs are refused before any CUDA call."""
import ctypes as C
import os
import re

from dd3d_b200 import lib

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
GRAPH_FUNCTIONS = ("dd3d_graph_create", "dd3d_graph_launch", "dd3d_graph_destroy", "dd3d_graph_kernel_nodes",
                   "dd3d_graph_programmatic_edges")
DD3D_ERR_INVALID = -1


def test_header_declares_the_graph_functions():
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        header = f.read()
    assert re.search(r"typedef\s+struct\s+dd3d_graph_t\s*\*\s*dd3d_graph\s*;", header)
    for name in GRAPH_FUNCTIONS:
        assert re.search(r"\b(int|void)\s+" + name + r"\s*\(", header), name


def test_library_exports_the_graph_functions():
    L = lib.load()
    for name in GRAPH_FUNCTIONS:
        assert name in lib.SIGNATURES
        assert getattr(L, name) is not None


def test_null_handle_and_graph_are_refused():
    L = lib.load()
    g = C.c_void_p(1)
    dummy = C.c_void_p(16)
    assert L.dd3d_graph_create(None, dummy, lib.IMG_U8, dummy, dummy, dummy, dummy, None, C.byref(g)) == DD3D_ERR_INVALID
    assert g.value is None  # *out is cleared on every refusal
    assert L.dd3d_graph_launch(None, None) == DD3D_ERR_INVALID
    assert L.dd3d_graph_kernel_nodes(None) == DD3D_ERR_INVALID
    assert L.dd3d_graph_programmatic_edges(None) == DD3D_ERR_INVALID


def test_missing_buffers_are_refused():
    L = lib.load()
    g = C.c_void_p(1)
    dummy = C.c_void_p(16)
    for i in range(5):
        bufs = [dummy] * 5
        bufs[i] = None
        assert L.dd3d_graph_create(None, bufs[0], lib.IMG_U8, bufs[1], bufs[2], bufs[3], bufs[4], None,
                                   C.byref(g)) == DD3D_ERR_INVALID
    assert L.dd3d_graph_create(None, dummy, lib.IMG_U8, dummy, dummy, dummy, dummy, None, None) == DD3D_ERR_INVALID


def test_destroy_null_graph_is_a_no_op():
    lib.load().dd3d_graph_destroy(None)
