"""Host side of the NuscenesDD3D sample aggregation as an engine step: the kernel-path rule, the extended packed layout,
the C ABI exports, the errors raised before any device work, and a world-size-2 gloo gather of the extended buffer in one
collective."""
import os
import re
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dd3d_b200 import lib
from dd3d_b200.gather import DetectionGatherer, PackedDetections, split_gathered

NEW_SYMBOLS = ("dd3d_set_sample_aggregate", "dd3d_set_groups", "dd3d_set_host_groups", "dd3d_set_global_out",
               "dd3d_set_host_global_out", "dd3d_sample_aggregate_path", "dd3d_packed_bytes_global")
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dd3d_b200.h")


def _nusc_cfg(do_nms=True, post_nms_topk=None):
    from dd3d_b200.config import get_cfg
    cfg = get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D")
    cfg.DD3D.INFERENCE.DO_NMS = do_nms
    if post_nms_topk is not None:
        cfg.DD3D.FCOS2D.INFERENCE.POST_NMS_TOPK = post_nms_topk
    return cfg


@pytest.mark.parametrize("do_nms,post,expect", [
    (True, None, lib.AGG_PATH_ONE_CTA),    # the shipped nuScenes config (POST_NMS_TOPK 100)
    (True, 1, lib.AGG_PATH_ONE_CTA),
    (True, 128, lib.AGG_PATH_ONE_CTA),     # 6 x 128 = 768: the one-CTA group still holds a sample
    (True, 129, lib.AGG_PATH_BLOCKED),
    (True, 300, lib.AGG_PATH_BLOCKED),
    (True, 1000, lib.AGG_PATH_BLOCKED),
    (True, 0, lib.AGG_PATH_BLOCKED),       # no post-NMS top-k: every 2-D NMS survivor
    (False, None, lib.AGG_PATH_BLOCKED),   # no 2-D NMS: L * PRE_NMS_TOPK candidates per image
    (False, 100, lib.AGG_PATH_BLOCKED),
])
def test_path_rule(do_nms, post, expect):
    L = lib.load()
    desc = lib.desc_from_cfg(_nusc_cfg(do_nms, post))
    assert L.dd3d_sample_aggregate_path(desc) == expect
    # a caller-sized output buffer beyond the one-CTA kernel's 256 slots takes the blocked path
    if expect == lib.AGG_PATH_ONE_CTA:
        desc.out_cap = 257
        assert L.dd3d_sample_aggregate_path(desc) == lib.AGG_PATH_BLOCKED
    assert L.dd3d_sample_aggregate_path(None) < 0


@pytest.mark.parametrize("B,cap", [(1, 128), (6, 128), (30, 128), (18, 160), (7, 5750), (30, 5750)])
def test_extended_packed_layout(B, cap):
    L = lib.load()
    base, ext = int(L.dd3d_packed_bytes(B, cap)), int(L.dd3d_packed_bytes_global(B, cap))
    assert PackedDetections.packed_bytes(B, cap) == base
    assert PackedDetections.packed_bytes(B, cap, with_global=True) == ext
    assert ext == base + (B * cap * 40 + 255) // 256 * 256
    p, q = PackedDetections(B, cap, "cpu"), PackedDetections(B, cap, "cpu", with_global=True)
    assert q.global_rows.shape == (B, cap, 10) and p.global_rows is None
    # the first three parts sit at the same byte offsets in both layouts
    for a, b in ((p.out, q.out), (p.counts, q.counts), (p.flags, q.flags)):
        assert a.data_ptr() - p.buf.data_ptr() == b.data_ptr() - q.buf.data_ptr()
        assert a.shape == b.shape
    assert q.global_rows.data_ptr() - q.buf.data_ptr() == base
    q.global_rows[B - 1, cap - 1, 9] = 7.0
    q.flags[0] = 5
    assert q.buf[base:].view(torch.float32)[B * cap * 10 - 1] == 7.0
    assert q.buf[B * cap * 96:base].view(torch.int32)[B] == 5
    assert L.dd3d_packed_bytes_global(0, cap) < 0 and L.dd3d_packed_bytes_global(B, 0) < 0


def test_new_abi_exports():
    L = lib.load()
    header = open(HEADER).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\b" + name + r"\(", header), name
        assert name in lib.SIGNATURES, name
        getattr(L, name)  # AttributeError if the library lacks it
    # a NULL handle is refused without touching a device
    assert L.dd3d_set_sample_aggregate(None, 1, 0.3, 500) == -1
    assert L.dd3d_set_groups(None, None, 0) == -1
    assert L.dd3d_set_host_groups(None, 0, None, 1) == -1
    assert L.dd3d_set_global_out(None, None) == -1
    assert L.dd3d_set_host_global_out(None, 0, None) == -1


def _model(**over):
    from dd3d_b200.meta_arch import NuscenesDD3DB200
    m = NuscenesDD3DB200(_nusc_cfg())
    for k, v in over.items():
        setattr(m, k, v)
    return m


def _inputs(tokens, out_sizes=None):
    from dd3d_b200.synthetic import make_nusc_inputs
    inputs = make_nusc_inputs(2, 64, 96, 500.0)[:len(tokens)]
    for i, (x, t) in enumerate(zip(inputs, tokens)):
        x["sample_token"] = t
        x["height"], x["width"] = out_sizes[i] if out_sizes else (128, 192)
        x["image_hwc"] = x["image"].permute(1, 2, 0).contiguous().numpy()
    return inputs


@pytest.mark.parametrize("path", ["forward", "forward_host", "submit_host", "forward_raw"])
def test_errors_before_device_work(path):
    """get_group_idxs's ValueError and the one-output-size assert come before the engine exists (on a machine without a
    GPU any device work would raise RuntimeError instead)."""
    m = _model()
    call = getattr(m, path)
    with pytest.raises(ValueError, match="Group sizes"):
        call(_inputs(["a"] * 5 + ["b"] * 7))
    if path != "forward_raw":  # the raw path's output sizes are the images' own (one size per call here)
        sizes = [(128, 192)] * 11 + [(130, 192)]
        with pytest.raises(AssertionError, match="output size"):
            call(_inputs(["a"] * 6 + ["b"] * 6, sizes))
    assert m._handle is None
    # the test hook off: no aggregation, so no group check -- the call gets as far as the missing device / weights
    m.sample_aggregate_in_inference = False
    with pytest.raises(RuntimeError):
        call(_inputs(["a"] * 5 + ["b"] * 7))


def test_raw_path_output_size_check():
    m = _model()
    inputs = _inputs(["a"] * 6)
    inputs[3]["image_hwc"] = np.zeros((60, 96, 3), dtype=np.uint8)
    with pytest.raises(AssertionError, match="output size"):
        m.forward_raw(inputs)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _fake(rank, B, cap):
    g = torch.Generator().manual_seed(200 + rank)
    return (torch.randn(B, cap, 24, generator=g), torch.randint(0, cap + 1, (B, ), generator=g, dtype=torch.int32),
            torch.randn(B, cap, 10, generator=g))


def _worker(rank, world, port, B, cap, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out, counts, glob = _fake(rank, B, cap)
    calls = []
    orig = dist.all_gather_into_tensor
    dist.all_gather_into_tensor = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    packed = PackedDetections(B, cap, "cpu", with_global=True)
    packed.out.copy_(out)
    packed.counts.copy_(counts)
    packed.flags.fill_(rank + 3)
    packed.global_rows.copy_(glob)
    gat = DetectionGatherer(B, cap, "cpu", with_global=True)
    g_out, g_cnt, g_flags, g_glob = gat.gather(packed)
    dist.all_gather_into_tensor = orig
    ok = len(calls) == 1 and g_flags.tolist() == [3, 4]
    for r in range(world):
        o, c, gl = _fake(r, B, cap)
        sl = slice(r * B, (r + 1) * B)
        ok &= torch.equal(g_out[sl], o) and torch.equal(g_cnt[sl], c) and torch.equal(g_glob[sl], gl)
    # the same bytes through split_gathered of a caller-held receive buffer
    recv = gat.new_recv()
    dist.all_gather_into_tensor(recv, packed.buf)
    s_out, s_cnt, s_flags, s_glob = split_gathered(recv, world, B, cap, with_global=True)
    ok &= torch.equal(s_out, g_out) and torch.equal(s_glob, g_glob) and torch.equal(s_cnt, g_cnt)
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_extended_gather_world2_gloo():
    world, B, cap = 2, 6, 8
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, B, cap, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert res == {0: True, 1: True}
