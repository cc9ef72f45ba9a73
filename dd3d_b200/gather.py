"""Whole-batch gather of packed detections across ranks (SURVEY.md 8e): ONE collective per evaluated batch.

Replaces the reference's `d2_comm.gather` of pickled python lists (kitti_3d_evaluator.py:152-164, nuscenes_evaluator.py:255).
Every rank owns one PACKED buffer (include/dd3d_b200.h dd3d_packed_bytes):

    dd3d_det[B][out_cap] | int32 counts[B] | int32 flags | pad to 256 B

whose first two parts are handed to dd3d_forward as d_out / d_counts, so the detections, their counts and the overflow
flags travel in a single fixed-size all-gather.  NuscenesDD3D uses the extended layout (dd3d_packed_bytes_global), the same
three parts at the same offsets followed by

    float global[B][out_cap][10] | pad to 256 B

the pred_boxes3d_global rows the engine's sample aggregation writes (dd3d_set_global_out), in the same collective:
  * on GPUs through the C ABI (dd3d_comm_* / dd3d_allgather = ncclAllGather, NCCL resolved at run time), on a SIDE stream
    ordered after the producing forward by an event -- the 295 KB exchange of batch k overlaps the forward of batch k+1 and
    no host synchronisation happens per step;
  * on CPU tensors through torch.distributed (gloo) -- the world-size-2 tests of the host logic.
Images are sharded by batch, rank r owns global images [r*B, (r+1)*B).
"""
import ctypes as C

import torch
import torch.distributed as dist

from . import lib as _lib


class PackedDetections:
    """One packed per-rank buffer (uint8 storage) with typed views: .out [B, cap, 24] fp32, .counts [B] int32,
    .flags [1] int32 and, with with_global, .global_rows [B, cap, 10] fp32 (all aliases of .buf)."""
    def __init__(self, B, cap, device, buf=None, with_global=False):
        self.B, self.cap, self.with_global = int(B), int(cap), bool(with_global)
        self.nbytes = self.packed_bytes(B, cap, with_global)
        self.buf = buf if buf is not None else torch.zeros(self.nbytes, dtype=torch.uint8, device=device)
        assert self.buf.numel() == self.nbytes and self.buf.dtype == torch.uint8
        det_bytes = self.B * self.cap * _lib.DET_WORDS * 4
        self.out = self.buf[:det_bytes].view(torch.float32).view(self.B, self.cap, _lib.DET_WORDS)
        head = self.packed_bytes(B, cap)
        tail = self.buf[det_bytes:head].view(torch.int32)
        self.counts = tail[:self.B]
        self.flags = tail[self.B:self.B + 1]
        self.global_rows = None
        if self.with_global:
            glob_bytes = self.B * self.cap * _lib.GLOBAL_WORDS * 4
            self.global_rows = self.buf[head:head + glob_bytes].view(torch.float32).view(self.B, self.cap, _lib.GLOBAL_WORDS)

    @staticmethod
    def packed_bytes(B, cap, with_global=False):
        """== dd3d_packed_bytes, or dd3d_packed_bytes_global with with_global (checked in the gather tests)."""
        det = int(B) * int(cap) * _lib.DET_WORDS * 4
        n = det + ((int(B) + 1) * 4 + 255) // 256 * 256
        if with_global:
            n += (int(B) * int(cap) * _lib.GLOBAL_WORDS * 4 + 255) // 256 * 256
        return n


def split_gathered(g_buf, world, B, cap, with_global=False):
    """[world * packed_bytes] uint8 -> ([world*B, cap, 24] fp32, [world*B] int32 counts, [world] int32 flags), and with
    with_global the [world*B, cap, 10] fp32 global rows as a fourth element."""
    n = PackedDetections.packed_bytes(B, cap, with_global)
    parts = [PackedDetections(B, cap, g_buf.device, buf=g_buf[r * n:(r + 1) * n], with_global=with_global)
             for r in range(world)]
    res = (torch.cat([p.out for p in parts], 0), torch.cat([p.counts for p in parts], 0),
           torch.cat([p.flags for p in parts], 0))
    if with_global:
        res += (torch.cat([p.global_rows for p in parts], 0), )
    return res


def unpack(g_out, g_cnt):
    """Per-image list of [n_i, 24] views in global image order."""
    return [g_out[i, :int(n)] for i, n in enumerate(g_cnt.tolist())]


class DetectionGatherer:
    """All-gather of PackedDetections buffers.  device "cuda": NCCL through the C ABI on a side stream; "cpu": gloo.
    with_global: the extended NuscenesDD3D layout, whose global rows travel in the same single collective."""
    def __init__(self, B, cap, device, rank=None, world=None, group=None, with_global=False):
        self.B, self.cap, self.device, self.group = int(B), int(cap), torch.device(device), group
        self.with_global = bool(with_global)
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world = dist.get_world_size(group) if world is None else world
        self.nbytes = PackedDetections.packed_bytes(B, cap, with_global)
        self.comm = None
        self.side = None
        if self.device.type == "cuda":
            L = _lib.load()
            uid = torch.zeros(128, dtype=torch.uint8)
            if self.rank == 0:
                if L.dd3d_comm_unique_id(C.c_void_p(uid.data_ptr())) != 0:
                    raise RuntimeError("dd3d_comm_unique_id: " + (L.dd3d_comm_last_error() or b"").decode())
            # the 128-byte NCCL id travels over the existing process group (any backend)
            box = [uid.tolist()]
            dist.broadcast_object_list(box, src=0, group=group)
            uid = torch.tensor(box[0], dtype=torch.uint8)
            comm = C.c_void_p()
            with torch.cuda.device(self.device):
                st = L.dd3d_comm_create(C.c_void_p(uid.data_ptr()), self.rank, self.world, C.byref(comm))
                if st != 0:
                    raise RuntimeError("dd3d_comm_create: " + (L.dd3d_comm_last_error() or b"").decode())
                self.side = torch.cuda.Stream(self.device)
            self.comm = comm

    def new_recv(self):
        return torch.zeros(self.world * self.nbytes, dtype=torch.uint8, device=self.device)

    def gather_async(self, packed, recv, stream=None):
        """Enqueue the all-gather of `packed` into `recv`.  CUDA: ordered after everything already enqueued on `stream`
        (default: the current stream), executed on the side stream; returns an event that fires when `recv` is complete and
        `packed` may be overwritten.  CPU: blocking; returns None."""
        if self.device.type != "cuda":
            dist.all_gather_into_tensor(recv, packed.buf, group=self.group)
            return None
        L = _lib.load()
        stream = stream or torch.cuda.current_stream(self.device)
        ready = torch.cuda.Event()
        ready.record(stream)
        self.side.wait_event(ready)
        st = L.dd3d_allgather(self.comm, C.c_void_p(packed.buf.data_ptr()), C.c_void_p(recv.data_ptr()), self.nbytes,
                              C.c_void_p(self.side.cuda_stream))
        if st != 0:
            raise RuntimeError("dd3d_allgather: " + (L.dd3d_comm_last_error() or b"").decode())
        done = torch.cuda.Event()
        done.record(self.side)
        return done

    def gather(self, packed, recv=None):
        """Blocking convenience: returns (g_out, g_counts, g_flags) of all ranks, and g_global with with_global."""
        assert packed.nbytes == self.nbytes, "packed buffer layout differs from the gatherer's"
        recv = recv if recv is not None else self.new_recv()
        done = self.gather_async(packed, recv)
        if done is not None:
            done.synchronize()
        return split_gathered(recv, self.world, self.B, self.cap, self.with_global)

    def close(self):
        if self.comm is not None:
            _lib.load().dd3d_comm_destroy(self.comm)
            self.comm = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def all_gather_detections(out, counts, group=None):
    """Compatibility helper for callers holding separate (out, counts) tensors: packs them into one buffer and runs ONE
    collective.  Returns ([world*B, cap, 24], [world*B]) on every rank."""
    B, cap = out.shape[0], out.shape[1]
    packed = PackedDetections(B, cap, out.device)
    packed.out.copy_(out)
    packed.counts.copy_(counts)
    g = DetectionGatherer(B, cap, out.device, group=group)
    try:
        g_out, g_cnt, _ = g.gather(packed)
    finally:
        g.close()
    return g_out, g_cnt
