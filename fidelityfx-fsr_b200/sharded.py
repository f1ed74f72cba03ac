"""Row-slab sharding of the EASU+RCAS path across the GPUs of one box (SURVEY.md §8(e)).

The reference has no multi-GPU path; this is new.  Every output pixel depends on a bounded input
neighbourhood, so the OUTPUT is cut into G contiguous row slabs, rank k owns input rows
[k*inH/G, (k+1)*inH/G) and needs a few more rows above/below (the EASU footprint of its output slab
extended by one output row each side, so that RCAS's +-1-row taps need no second exchange).
The only communication is that halo, between neighbouring ranks; there is no reduction and a 1-GPU run issues
no communication at all.  Two data planes move it:

  halo="p2p"   (default on CUDA) the C ABI's fsr1_shard_* (csrc/fsr1_shard.cu): every rank pushes its edge rows
               straight into the neighbour's window with 128-bit NVLink stores from a small kernel, flow-controlled by
               sequence numbers in device memory (CUDA IPC between the ranks' processes).  No NCCL call, no host
               synchronisation per frame; RCAS of frame i overlaps EASU of frame i+1 on every rank.
               torch.distributed is used ONCE, to gather the 64-byte IPC handles.
  halo="nccl"  torch.distributed point-to-point (ncclSend/ncclRecv in one group per frame) into the edge rows of the
               rank's window tensor; works on any backend (gloo with CPU tensors in the tests).

SlabPlan is pure integer geometry (unit-tested on CPU and against the C ABI's own plan).
"""
import ctypes
import math

import numpy as np

from . import _lib, api


def _cell(o, scale, offset):
    """floor(o*scale+offset) in the kernels' float arithmetic (mul and add rounded separately)."""
    return int(math.floor(np.float32(np.float32(np.float32(o) * np.float32(scale)) + np.float32(offset))))


class SlabPlan:
    def __init__(self, in_h, out_h, world, easu_con):
        self.in_h, self.out_h, self.world = int(in_h), int(out_h), int(world)
        if self.world < 1 or self.world > self.in_h or self.world > self.out_h:
            raise ValueError("row-slab plan needs 1 <= world <= rows (no empty slabs): world=%d in_h=%d out_h=%d"
                             % (self.world, self.in_h, self.out_h))
        self.scale = np.array([easu_con[1]], dtype=np.uint32).view(np.float32)[0]
        self.offset = np.array([easu_con[3]], dtype=np.uint32).view(np.float32)[0]

    def out_rows(self, rank):
        """Output rows [y0,y1) of this rank's slab."""
        return rank * self.out_h // self.world, (rank + 1) * self.out_h // self.world

    def easu_rows(self, rank):
        """EASU is run for the slab plus a one-row apron (what RCAS reads)."""
        y0, y1 = self.out_rows(rank)
        return max(y0 - 1, 0), min(y1 + 1, self.out_h)

    def owned_in_rows(self, rank):
        return rank * self.in_h // self.world, (rank + 1) * self.in_h // self.world

    def needed_in_rows(self, rank):
        """Input rows [r0,r1) the rank's EASU pass reads (clamped to the image)."""
        e0, e1 = self.easu_rows(rank)
        lo = _cell(e0, self.scale, self.offset) - 1
        hi = _cell(e1 - 1, self.scale, self.offset) + 2
        lo = min(max(lo, 0), self.in_h - 1)
        hi = min(max(hi, 0), self.in_h - 1)
        return lo, hi + 1

    def window_rows(self, rank):
        """Input rows resident on the rank: its own slab plus the halo."""
        (n0, n1), (o0, o1) = self.needed_in_rows(rank), self.owned_in_rows(rank)
        return min(n0, o0), max(n1, o1)

    def transfers(self, rank):
        """(sends, recvs): lists of (peer, first_row, end_row) in logical input rows."""
        sends, recvs = [], []
        own0, own1 = self.owned_in_rows(rank)
        need0, need1 = self.needed_in_rows(rank)
        for peer in range(self.world):
            if peer == rank:
                continue
            p_own0, p_own1 = self.owned_in_rows(peer)
            p_need0, p_need1 = self.needed_in_rows(peer)
            a, b = max(own0, p_need0), min(own1, p_need1)      # my rows the peer needs
            if b > a:
                sends.append((peer, a, b))
            a, b = max(p_own0, need0), min(p_own1, need1)      # the peer's rows I need
            if b > a:
                recvs.append((peer, a, b))
        return sends, recvs

    def halo_bytes(self, rank, width, bytes_per_pixel):
        return sum((b - a) * width * bytes_per_pixel for _, a, b in self.transfers(rank)[1])


def exchange_halo(plan, rank, owned, window, dist=None):
    """Fill `window` (rows needed_in_rows(rank)) from `owned` (rows owned_in_rows(rank)) and the peers.

    `owned` may be a view INTO `window`: then nothing is copied locally and only the halo rows move.
    Works on any backend: gloo with CPU tensors (tests) or nccl with CUDA tensors.
    """
    own0, own1 = plan.owned_in_rows(rank)
    need0, need1 = plan.needed_in_rows(rank)
    a, b = max(own0, need0), min(own1, need1)
    if b > a and owned[a - own0:a - own0 + 1].data_ptr() != window[a - need0:a - need0 + 1].data_ptr():
        window[a - need0:b - need0].copy_(owned[a - own0:b - own0])
    sends, recvs = plan.transfers(rank)
    if not sends and not recvs:
        return 0
    if dist is None:
        import torch.distributed as dist
    ops = []
    for peer, r0, r1 in sends:
        ops.append(dist.P2POp(dist.isend, owned[r0 - own0:r1 - own0], peer))
    for peer, r0, r1 in recvs:
        ops.append(dist.P2POp(dist.irecv, window[r0 - need0:r1 - need0], peer))
    for req in dist.batch_isend_irecv(ops):
        req.wait()
    return len(ops)


def exchange_halo_many(plan, rank, frames, dist=None):
    """The halo exchange of SEVERAL frames in ONE batched group.  `frames` is a list of (owned, window) pairs as
    for exchange_halo; every rank must pass its frames in the same order.  Returns the number of point-to-point ops."""
    own0, own1 = plan.owned_in_rows(rank)
    need0, need1 = plan.needed_in_rows(rank)
    a, b = max(own0, need0), min(own1, need1)
    sends, recvs = plan.transfers(rank)
    if dist is None:
        import torch.distributed as dist
    ops = []
    for owned, window in frames:
        if b > a and owned[a - own0:a - own0 + 1].data_ptr() != window[a - need0:a - need0 + 1].data_ptr():
            window[a - need0:b - need0].copy_(owned[a - own0:b - own0])
        for peer, r0, r1 in sends:
            ops.append(dist.P2POp(dist.isend, owned[r0 - own0:r1 - own0], peer))
        for peer, r0, r1 in recvs:
            ops.append(dist.P2POp(dist.irecv, window[r0 - need0:r1 - need0], peer))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return len(ops)


class _DevBuf:
    """A raw device allocation described through __cuda_array_interface__ (zero-copy torch view of C-ABI-owned memory)."""

    def __init__(self, ptr, shape, strides, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "strides": tuple(strides), "typestr": typestr,
                                         "data": (int(ptr), False), "version": 2}


def _tensor_of(img, device):
    """torch view [rows, width, 4] of an fsr1_image owned by the library ([rows, width] int32 for RGB10A2_UNORM and R11G11B10_FLOAT, as
    api.image takes)."""
    import torch
    if img.format in (_lib.FORMAT_RGB10A2_UNORM, _lib.FORMAT_R11G11B10_FLOAT):
        return torch.as_tensor(_DevBuf(img.data, (img.rows, img.width), (img.pitch_bytes, 4), "<i4"), device=device)
    es, typestr = {_lib.FORMAT_RGBA16F: (2, "<f2"), _lib.FORMAT_RGBA32F: (4, "<f4"), _lib.FORMAT_RGBA8_UNORM: (1, "|u1")}[img.format]
    return torch.as_tensor(_DevBuf(img.data, (img.rows, img.width, 4), (img.pitch_bytes, 4 * es, es), typestr), device=device)


class ShardedUpscaler:
    """One instance per rank (one process per GPU): the rank's share of a ring of `slots` frames.

    Per frame: write the rank's input rows into input(slot), submit(slot), then wait(slot) before reading output(slot).
    All ranks construct with the same arguments and submit slots in the same order.
    `owned` / `out` are slot 0's tensors; upscale() is the one-frame convenience over slot 0.
    halo="p2p" with world > 1 gathers the ranks' CUDA IPC handles through torch.distributed in the constructor (a collective:
    every rank constructs at the same point); attach=False skips that for ranks living in one process (attach_local).
    dynamic=True (p2p only): in_w x in_h is the input resource, the largest render size; frame(slot, render_w, render_h) gives the
    next use of a slot its own render size and sharpness (FSR1_SHARD_DYNAMIC, fsr1_shard_frame) before its rows are written.
    srtm_inverse / grain, amount / tepd_bits, dither (p2p only): the display steps of api.upscale_post run inside every frame
    (fsr1_shard_create_post), so output(slot) is the display image's rows: uint8 [rows, W, 4] with tepd_bits 8, int32 [rows, W] with 10,
    float16 [rows, W, 4] otherwise.  post(slot, frame=...) describes the next use of a slot (fsr1_shard_post).  The grain / dither
    tiles are device tensors the ranks read while frames are in flight; this object keeps a reference to the ones each slot uses.
    in_format=FORMAT_R11G11B10_FLOAT (p2p only): the input windows hold R11G11B10_FLOAT codes, int32 [rows, W] (4 B/px: the windows and
    the halo are half the size of RGBA16F ones); the output slabs are float16 [rows, W, 4] (or the TEPD format).  `dtype` is ignored then.
    """

    def __init__(self, in_w, in_h, out_w, out_h, world, rank, sharpness=0.25, dtype=None, device=None, flags=0, slots=1,
                 halo=None, one_stream=False, group=None, skip_halo=False, attach=True, trace=False, dynamic=False,
                 srtm_inverse=False, grain=None, amount=0.0, tepd_bits=0, dither=None, in_format=None):
        import torch
        self.rank, self.world, self.slots = int(rank), int(world), int(slots)
        self.in_w, self.in_h, self.out_w, self.out_h = in_w, in_h, out_w, out_h
        self.sharpness, self.dynamic = sharpness, bool(dynamic)
        self._post_args = (bool(srtm_inverse), grain, amount, tepd_bits, dither)
        self.has_post = bool(srtm_inverse) or grain is not None or tepd_bits != 0
        self.econ = api.easu_con(in_w, in_h, in_w, in_h, out_w, out_h)
        self.rcon = api.rcas_con(sharpness)
        self.plan = SlabPlan(in_h, out_h, world, self.econ)
        self.flags, self.group = flags, group
        dtype = dtype or torch.float16
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        if halo is None:
            halo = "p2p" if self.device.type == "cuda" else "nccl"
        if halo not in ("p2p", "nccl"):
            raise ValueError("halo must be 'p2p' or 'nccl'")
        if self.dynamic and halo != "p2p":
            raise ValueError("dynamic=True needs halo='p2p' (the per-frame plan lives in the C ABI's shard)")
        if in_format not in (None, _lib.FORMAT_R11G11B10_FLOAT):
            raise ValueError("in_format: None (from dtype) or FORMAT_R11G11B10_FLOAT")
        if in_format is not None and halo != "p2p":
            raise ValueError("in_format=FORMAT_R11G11B10_FLOAT needs halo='p2p' (its kernels run inside the C ABI's shard)")
        self.in_format = in_format
        if self.has_post and halo != "p2p":
            raise ValueError("display steps (srtm_inverse, grain, tepd_bits) need halo='p2p' (they run inside the C ABI's shard)")
        self.halo_mode = halo
        self._win0 = self.plan.window_rows(rank)[0]
        self._shard = None
        if halo == "p2p":
            self._init_p2p(sharpness, dtype, one_stream, skip_halo, attach, trace)
        else:
            self._init_nccl(dtype)
        self.owned, self.out, self.window = self.inputs[0], self.outputs[0], self.windows[0]

    # ------------------------------------------------------------------------------------------ p2p (C ABI) data plane
    def _init_p2p(self, sharpness, dtype, one_stream, skip_halo=False, attach=True, trace=False):
        import torch
        L = _lib.lib()
        if self.in_format is not None:
            fmt = self.in_format
        else:
            fmt = {torch.float16: _lib.FORMAT_RGBA16F, torch.float32: _lib.FORMAT_RGBA32F, torch.uint8: _lib.FORMAT_RGBA8_UNORM}[dtype]
        srtm_inverse, grain, amount, tepd_bits, dither = self._post_args
        post, keep = api._post(srtm_inverse, grain, amount, tepd_bits, dither, 0)
        mid_fmt = _lib.FORMAT_RGBA16F if fmt == _lib.FORMAT_R11G11B10_FLOAT else fmt   # EASU's output format
        out_fmt = {0: mid_fmt, 8: _lib.FORMAT_RGBA8_UNORM, 10: _lib.FORMAT_RGB10A2_UNORM}[tepd_bits]
        self._tiles = [(grain, dither)] * self.slots     # the tiles each slot's next use reads
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(L.fsr1_shard_create_post(ctypes.byref(h), self.in_w, self.in_h, self.out_w, self.out_h, fmt, out_fmt,
                                                ctypes.byref(post) if self.has_post else None, self.world, self.rank,
                                                self.slots, ctypes.c_float(sharpness),
                                                self.flags | (_lib.SHARD_ONE_STREAM if one_stream else 0) | (_lib.SHARD_SKIP_HALO if skip_halo else 0) | (_lib.SHARD_TRACE if trace else 0)
                                                | (_lib.SHARD_DYNAMIC if self.dynamic else 0)))
        del keep
        self._shard = h
        info = _lib.ShardInfo()
        _lib.check(L.fsr1_shard_geometry(h, ctypes.byref(info)))
        self.info = info
        plan, r = self.plan, self.rank
        assert (info.out_row0, info.out_row1) == plan.out_rows(r) and (info.owned_row0, info.owned_row1) == plan.owned_in_rows(r)
        assert (info.needed_row0, info.needed_row1) == plan.needed_in_rows(r) and (info.window_row0, info.window_row1) == plan.window_rows(r)
        self.inputs, self.outputs, self.windows = [], [], []
        for s in range(self.slots):
            a, w, b = _lib.Image(), _lib.Image(), _lib.Image()
            _lib.check(L.fsr1_shard_input(h, s, ctypes.byref(a)))
            _lib.check(L.fsr1_shard_window(h, s, ctypes.byref(w)))
            _lib.check(L.fsr1_shard_output(h, s, ctypes.byref(b)))
            self.inputs.append(_tensor_of(a, self.device))
            self.windows.append(_tensor_of(w, self.device))
            self.outputs.append(_tensor_of(b, self.device))
        if self.world > 1 and attach and not skip_halo:   # attach=False: the caller attaches (attach_local, several ranks in one process)
            self._attach_ipc()

    def _attach_ipc(self):
        """Gather every rank's 64-byte CUDA IPC handle (the only use of torch.distributed on this path) and map the
        neighbours' arenas."""
        import torch
        import torch.distributed as dist
        L = _lib.lib()
        mine = (ctypes.c_ubyte * _lib.SHARD_HANDLE_BYTES)()
        _lib.check(L.fsr1_shard_export(self._shard, mine))
        backend = dist.get_backend(self.group)
        dev = self.device if backend == "nccl" else torch.device("cpu")
        t = torch.tensor(list(bytes(mine)), dtype=torch.uint8, device=dev)
        gathered = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(gathered, t, group=self.group)
        blob = b"".join(bytes(g.cpu().numpy().tobytes()) for g in gathered)
        _lib.check(L.fsr1_shard_attach(self._shard, blob, self.world))
        dist.barrier(group=self.group)

    def attach_local(self, up=None, down=None):
        """Several ranks inside ONE process (one thread driving several devices, or a single-GPU test): neighbours by
        object instead of by IPC handle."""
        _lib.check(_lib.lib().fsr1_shard_attach_local(self._shard, up._shard if up is not None else None,
                                                      down._shard if down is not None else None))

    # ------------------------------------------------------------------------------------------ nccl / gloo data plane
    def _init_nccl(self, dtype):
        import torch
        plan, r = self.plan, self.rank
        (lo, hi), (o0, o1), (e0, e1), (y0, y1) = plan.window_rows(r), plan.owned_in_rows(r), plan.easu_rows(r), plan.out_rows(r)
        dev = self.device
        self.windows = [torch.zeros((hi - lo, self.in_w, 4), dtype=dtype, device=dev) for _ in range(self.slots)]
        self.inputs = [w[o0 - lo:o1 - lo] for w in self.windows]
        self.tmps = [torch.empty((e1 - e0, self.out_w, 4), dtype=dtype, device=dev) for _ in range(self.slots)]
        self.outputs = [torch.empty((y1 - y0, self.out_w, 4), dtype=dtype, device=dev) for _ in range(self.slots)]
        sends, recvs = plan.transfers(r)
        # halo transfers as views of each slot's window, built once: rows to send / receive per peer
        self._sends = [[(peer, w[a - lo:b - lo]) for peer, a, b in sends] for w in self.windows]
        self._recvs = [[(peer, w[a - lo:b - lo]) for peer, a, b in recvs] for w in self.windows]
        self._prepared = [None] * self.slots

    def _exchange(self, slot=0):
        """nccl mode: the slot's halo rows, one batched point-to-point group (every rank with a neighbour takes part)."""
        import torch.distributed as dist
        ops = [dist.P2POp(dist.isend, t, peer, group=self.group) for peer, t in self._sends[slot]]
        ops += [dist.P2POp(dist.irecv, t, peer, group=self.group) for peer, t in self._recvs[slot]]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        return len(ops)

    def exchange_many(self, slots):
        """nccl mode: the halos of several slots in ONE batched group (amortises the per-exchange launch cost)."""
        import torch.distributed as dist
        ops = []
        for s in slots:
            ops += [dist.P2POp(dist.isend, t, peer, group=self.group) for peer, t in self._sends[s]]
            ops += [dist.P2POp(dist.irecv, t, peer, group=self.group) for peer, t in self._recvs[s]]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        return len(ops)

    def _launch(self, slot=0, stream=None):
        """nccl mode: EASU (slab + apron) then RCAS on `stream`."""
        if self._prepared[slot] is None:
            plan, r = self.plan, self.rank
            e0, _ = plan.easu_rows(r)
            y0, y1 = plan.out_rows(r)
            self._prepared[slot] = api.PreparedUpscale(
                api.image(self.windows[slot], height=self.in_h, row0=self._win0), api.image(self.tmps[slot], height=self.out_h, row0=e0),
                api.image(self.outputs[slot], height=self.out_h, row0=y0), self.econ, self.rcon, y0=y0, y1=y1, flags=self.flags)
        self._prepared[slot].launch(stream)

    def frame(self, slot, render_w, render_h, sharpness=None):
        """dynamic=True: the next use of `slot` upscales the top-left render_w x render_h of the resource with `sharpness` (None: the
        constructor's).  Call it before writing the frame's rows; returns input(slot), the rank's owned rows of that frame
        ([rows, render_w, 4]).  Every rank describes the same use of a slot with the same arguments."""
        if not self.dynamic:
            raise ValueError("frame() needs a ShardedUpscaler constructed with dynamic=True")
        L = _lib.lib()
        sharp = self.sharpness if sharpness is None else sharpness
        _lib.check(L.fsr1_shard_frame(self._shard, slot, render_w, render_h, ctypes.c_float(sharp)))
        a, w = _lib.Image(), _lib.Image()
        _lib.check(L.fsr1_shard_input(self._shard, slot, ctypes.byref(a)))
        _lib.check(L.fsr1_shard_window(self._shard, slot, ctypes.byref(w)))
        plan, r = SlabPlan(render_h, self.out_h, self.world, api.easu_con(render_w, render_h, render_w, render_h, self.out_w, self.out_h)), self.rank
        assert (a.row0, a.row0 + a.rows) == plan.owned_in_rows(r) and (w.row0, w.row0 + w.rows) == plan.window_rows(r)
        assert (a.width, a.height, w.width, w.height) == (render_w, render_h, render_w, render_h)
        self.inputs[slot], self.windows[slot] = _tensor_of(a, self.device), _tensor_of(w, self.device)
        if slot == 0:
            self.owned, self.window = self.inputs[0], self.windows[0]
        return self.inputs[slot]

    def post(self, slot, frame=0, amount=None, grain=None, dither=None):
        """The display steps of the next use of `slot` (fsr1_shard_post): the TEPD `frame` of the positional dither, the LFGA amount and
        the tiles; None keeps the constructor's amount / grain / dither.  The steps themselves (srtm_inverse, LFGA, tepd_bits) are the
        constructor's."""
        if not self.has_post:
            raise ValueError("post() needs a ShardedUpscaler constructed with display steps (srtm_inverse, grain or tepd_bits)")
        srtm_inverse, grain0, amount0, tepd_bits, dither0 = self._post_args
        grain = grain0 if grain is None else grain
        dither = dither0 if dither is None else dither
        post, keep = api._post(srtm_inverse, grain, amount0 if amount is None else amount, tepd_bits, dither, frame)
        _lib.check(_lib.lib().fsr1_shard_post(self._shard, slot, ctypes.byref(post)))
        del keep
        self._tiles[slot] = (grain, dither)

    # ------------------------------------------------------------------------------------------ common
    def input(self, slot=0):
        return self.inputs[slot]

    def output(self, slot=0):
        return self.outputs[slot]

    def submit(self, slot=0, stream=None):
        """Upscale the frame whose rows are in input(slot); ordered after everything already on `stream`."""
        if self._shard is not None:
            rc = _lib.lib().fsr1_shard_submit(self._shard, slot, api._stream(stream))
            if rc:
                _lib.check(rc)
            return
        if self.world > 1:
            self._exchange(slot)
        self._launch(slot, stream)

    def wait(self, slot=0, stream=None):
        """Order `stream` after the slot's result (p2p: also after this rank's halo rows have left)."""
        if self._shard is not None:
            _lib.check(_lib.lib().fsr1_shard_wait(self._shard, slot, api._stream(stream)))

    def trace(self, max_frames=256):
        """p2p with trace=True: [n, 8] uint64 GPU timestamps (ns) of the last frames (see fsr1_shard_trace)."""
        import numpy as np
        buf = (ctypes.c_uint64 * (8 * max_frames))()
        n = ctypes.c_uint32()
        _lib.check(_lib.lib().fsr1_shard_trace(self._shard, buf, max_frames, ctypes.byref(n)))
        return np.frombuffer(buf, dtype=np.uint64).reshape(max_frames, 8)[:n.value].copy()

    def status(self):
        """p2p: raises if a neighbour's halo or credit timed out (call after a synchronize)."""
        if self._shard is not None:
            _lib.check(_lib.lib().fsr1_shard_status(self._shard))

    def upscale(self, owned_rows=None, stream=None):
        """One frame through slot 0: returns the rank's output slab (valid on `stream`)."""
        if owned_rows is not None and owned_rows.data_ptr() != self.owned.data_ptr():
            self.owned.copy_(owned_rows)
        self.submit(0, stream)
        self.wait(0, stream)
        return self.out

    def close(self):
        if self._shard is not None:
            self.inputs = self.outputs = self.windows = []
            self.owned = self.out = self.window = None
            _lib.lib().fsr1_shard_destroy(self._shard)
            self._shard = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
