"""Clip-level data parallelism: clips are independent units, so they shard across ranks with no
data-path collective; the ONLY collective is one all-gather of the output frames for the stitch.

One process per GPU (torchrun); ``nccl`` on GPUs, ``gloo`` in the CPU tests.

Round 2 (VERDICT r01 "Multi-GPU"):
* clips shard in contiguous BLOCKS (rank r owns clips [r*share, (r+1)*share)), so the all-gather lands in global clip
  order and the 637 MB transpose-reshape copy of the round-robin layout is gone;
* the stitch is asynchronous and double-buffered (``ClipStitcher``): the all-gather of step i runs on the
  communication stream while the forward of step i+1 computes;
* the payload can be fp32 (exact, default), fp16, or the uint8 frames test.py actually keeps
  (``((x + 1) / 2 * 255)`` truncated, test.py:168-169) — 2x / 4x fewer bytes over NVLink;
* on one NVLink / NVSwitch box the payload does not go through NCCL at all (``PeerStitcher``): every rank pushes its
  block of frames into the peers' landing buffers (CUDA IPC peer memory) with copy-engine DMA on a side stream and
  orders the pushes with flag words driven by stream memory operations — no kernel, no SM, so the persistent
  one-CTA-per-SM kernels of the next forward keep the whole chip while the exchange runs.  The peer path is the
  default because it cannot compete for SMs as payloads grow.
"""
import os

import torch
import torch.distributed as dist

PAYLOADS = ("fp32", "fp16", "uint8")


def init_from_env(backend=None):
    """Initialise torch.distributed from RANK / WORLD_SIZE / MASTER_* (torchrun). Returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
            dist.init_process_group(backend, rank=rank, world_size=world, device_id=torch.device("cuda", local_rank))
        else:
            dist.init_process_group(backend, rank=rank, world_size=world)
    return rank, world, local_rank


def padded_share(num_clips, world):
    """Clips per rank after padding to an equal share (all_gather needs equal sizes)."""
    return (num_clips + world - 1) // world


def shard_clips(num_clips, rank, world):
    """Clip ids owned by ``rank``: the contiguous block [rank*share, (rank+1)*share) clipped to num_clips.  Block
    (not round-robin) ownership makes the all-gather result already ordered by clip id."""
    share = padded_share(num_clips, world)
    return list(range(min(rank * share, num_clips), min((rank + 1) * share, num_clips)))


def encode_payload(pred, payload="fp32"):
    """What a rank sends into the stitch: fp32 predictions, their fp16 rounding, or test.py's uint8 frames
    (``(x + 1) / 2 * 255`` truncated like ``astype(np.uint8)``, test.py:168-169)."""
    if payload == "fp32":
        return pred.contiguous()
    if payload == "fp16":
        return pred.to(torch.float16).contiguous()
    if payload == "uint8":
        return ((pred + 1) / 2 * 255).clamp_(0, 255).to(torch.uint8).contiguous()
    raise ValueError(f"payload must be one of {PAYLOADS}")


class _Pending:
    """Handle of one in-flight stitch: ``wait()`` orders the CURRENT stream after the collective and returns the
    gathered (num_clips*T, 3, H, W) tensor (a view of one of the stitcher's two landing buffers: consume it before
    the stitch after next is started)."""

    def __init__(self, work, out, n_valid, keep):
        self.work, self.out, self.n_valid, self.keep = work, out, n_valid, keep

    def wait(self):
        if self.work is not None:
            self.work.wait()
            self.work = None
        self.keep = None
        return self.out[: self.n_valid]


class ClipStitcher:
    """Double-buffered asynchronous output stitch.  ``start(local_pred)`` launches the all-gather (NCCL: on the
    process group's communication stream, ordered after everything already enqueued on the current stream) and
    returns immediately, so the next forward overlaps it; ``_Pending.wait()`` joins."""

    def __init__(self, num_clips, frames_per_clip, rank, world, payload="fp32"):
        if payload not in PAYLOADS:
            raise ValueError(f"payload must be one of {PAYLOADS}")
        self.num_clips, self.T, self.rank, self.world, self.payload = num_clips, frames_per_clip, rank, world, payload
        self.share = padded_share(num_clips, world)
        self._bufs = [None, None]
        self._n = 0

    def start(self, local_pred):
        """local_pred: (share * T, 3, H, W) — this rank's clips in ``shard_clips`` order, zero-padded to the share."""
        n_valid = self.num_clips * self.T
        send = encode_payload(local_pred, self.payload)
        if self.world == 1:
            return _Pending(None, send, n_valid, None)
        if send.shape[0] != self.share * self.T:
            raise ValueError(f"local_pred has {send.shape[0]} frames, expected share*T = {self.share * self.T}")
        k = self._n & 1
        self._n += 1
        shape = (self.world * send.shape[0],) + tuple(send.shape[1:])
        buf = self._bufs[k]
        if buf is None or buf.shape != shape or buf.dtype != send.dtype or buf.device != send.device:
            buf = self._bufs[k] = torch.empty(shape, dtype=send.dtype, device=send.device)
        work = dist.all_gather_into_tensor(buf, send, async_op=True)
        return _Pending(work, buf, n_valid, send)


class _PendingPeer:
    """Handle of one in-flight peer-memory stitch (same contract as ``_Pending``)."""

    def __init__(self, done, out, n_valid, keep):
        self.done, self.out, self.n_valid, self.keep = done, out, n_valid, keep

    def wait(self):
        if self.done is not None:
            torch.cuda.current_stream().wait_event(self.done)
            self.done = None
        self.keep = None
        return self.out[: self.n_valid]


class _DevicePtr:
    """Minimal ``__cuda_array_interface__`` carrier: lets torch view a cudaMalloc'd landing buffer it does not own."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class PeerStitcher(ClipStitcher):
    """The stitch as copy-engine pushes into the peers' landing buffers (csrc/peer.cu); same ``start`` / ``wait``
    contract as ``ClipStitcher``.  Every rank owns two landing buffers and one block of 32-bit flag words
    (``may_write[r]``, ``landed[r]`` per peer r), all exported through CUDA IPC.  Step i (buffer k = i & 1), on the
    stitcher's side stream of rank me — DMA copies and stream memory operations only, no kernel, no SM:

        wait(event: pred computed and the readers of my buffer k have finished)
        for every peer p:  p.may_write[me] := i + 1          "you may overwrite my buffer k"
        for every peer p:  wait my.may_write[p] >= i + 1;  copy my block -> p.buffer[k][slot me];  p.landed[me] := i + 1
        copy my block -> my buffer k;  for every peer p: wait my.landed[p] >= i + 1

    Counters only grow, so a fast rank can run at most one buffer ahead of a slow one and never overwrites unread data."""

    def __init__(self, num_clips, frames_per_clip, rank, world, payload="fp32", group=None):
        super().__init__(num_clips, frames_per_clip, rank, world, payload)
        self.group = group
        self._stream = None
        self._local = [None, None, None]  # raw pointers: landing buffer 0, landing buffer 1, flag block
        self._remote = None               # [r] -> (buffer 0, buffer 1, flag block) of rank r as mapped here
        self._shape = None
        self._fallback = None             # ClipStitcher, if the peer-memory set-up failed on any rank

    # ---- one-time (per payload shape) collective setup: allocate, exchange IPC handles, map the peers' buffers.
    # Two votes (after allocating, after mapping): if ANY rank fails, every rank releases what it holds and the stitcher
    # degrades to the all-gather of ``ClipStitcher`` for good — never a rank-dependent choice, never a hang.
    def _setup(self, send):
        import ctypes
        import warnings

        from . import _lib
        lib = _lib.load()
        self.close()
        dev = send.device
        nbytes = self.world * send.numel() * send.element_size()
        shape = (self.world * send.shape[0],) + tuple(send.shape[1:])
        handles, err = [], None
        try:
            for k, size in enumerate((nbytes, nbytes, 2 * 4 * self.world)):
                ptr, h = ctypes.c_void_p(), ctypes.create_string_buffer(64)
                _lib.check(lib.e2f_peer_alloc(size, ctypes.byref(ptr), h), "e2f_peer_alloc")
                self._local[k] = ptr.value
                if k < 2:
                    self._bufs[k] = torch.as_tensor(_DevicePtr(ptr.value, nbytes), device=dev).view(send.dtype).view(shape)
                handles.append(bytes(h.raw))
        except Exception as exc:  # noqa: BLE001 - any failure here is answered by the collective fallback below
            err = repr(exc)
        everyone = [None] * self.world
        dist.all_gather_object(everyone, (err, handles), group=self.group)
        opened = []
        if all(e is None for e, _ in everyone):
            try:
                self._remote = []
                for r in range(self.world):
                    if r == self.rank:
                        self._remote.append(tuple(self._local))
                        continue
                    ptrs = []
                    for k in range(3):
                        ptr = ctypes.c_void_p()
                        _lib.check(lib.e2f_peer_open(everyone[r][1][k], ctypes.byref(ptr)), "e2f_peer_open")
                        ptrs.append(ptr.value)
                        opened.append(ptr.value)
                    self._remote.append(tuple(ptrs))
            except Exception as exc:  # noqa: BLE001
                err = repr(exc)
        else:
            err = err or "a peer failed to allocate its landing buffers"
        votes = [None] * self.world
        dist.all_gather_object(votes, err, group=self.group)
        if any(v is not None for v in votes):
            for ptr in opened:
                lib.e2f_peer_close(ptr)
            dist.barrier(group=self.group)                   # nobody frees memory a peer still has mapped
            for k in range(3):
                if self._local[k]:
                    lib.e2f_peer_free(self._local[k])
                self._local[k] = None
            self._bufs, self._remote = [None, None], None
            self._fallback = ClipStitcher(self.num_clips, self.T, self.rank, self.world, self.payload)
            if self.rank == 0:
                warnings.warn(f"PeerStitcher: peer-memory set-up failed ({[v for v in votes if v][0]}); using the all-gather")
            return
        self._shape, self._dtype, self._device = shape, send.dtype, dev
        self._n = 0                                          # flag words were zeroed with the allocation
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=dev)
        dist.barrier(group=self.group)                       # every rank has mapped every buffer before the first push

    def close(self):
        """Unmap the peers' buffers and free the local ones (collective: every rank must call it, or none)."""
        if self._shape is None:
            return
        from . import _lib
        lib = _lib.load()
        torch.cuda.synchronize(self._device)
        dist.barrier(group=self.group)                      # no rank is still pushing into buffers about to go away
        for r, ptrs in enumerate(self._remote):
            if r != self.rank:
                for ptr in ptrs:
                    lib.e2f_peer_close(ptr)
        dist.barrier(group=self.group)                      # nobody frees memory a peer still has mapped
        for k in range(3):
            lib.e2f_peer_free(self._local[k])
            self._local[k] = None
        self._bufs = [None, None]
        self._remote = None
        self._shape = None

    def start(self, local_pred):
        from . import _lib
        n_valid = self.num_clips * self.T
        send = encode_payload(local_pred, self.payload)
        if self.world == 1:
            return _Pending(None, send, n_valid, None)
        if send.shape[0] != self.share * self.T:
            raise ValueError(f"local_pred has {send.shape[0]} frames, expected share*T = {self.share * self.T}")
        shape = (self.world * send.shape[0],) + tuple(send.shape[1:])
        if self._fallback is None and (self._shape != shape or self._dtype != send.dtype or self._device != send.device):
            self._setup(send)
        if self._fallback is not None:
            return self._fallback.start(local_pred)
        k = self._n & 1
        self._n += 1
        seq = self._n & 0xFFFFFFFF                           # i + 1
        lib, me, W = _lib.load(), self.rank, self.world
        nbytes = send.numel() * send.element_size()
        ready = torch.cuda.Event()
        ready.record()                                      # pred computed; the readers of buffer k were enqueued before
        side = self._stream
        st = side.cuda_stream
        peers = [(me + 1 + j) % W for j in range(W - 1)]    # every rank starts at a different destination
        may_write = lambda owner, writer: self._remote[owner][2] + 4 * writer            # noqa: E731
        landed = lambda owner, writer: self._remote[owner][2] + 4 * (W + writer)         # noqa: E731
        with torch.cuda.stream(side):
            side.wait_event(ready)
            for p in peers:
                _lib.check(lib.e2f_peer_signal(may_write(p, me), seq, st), "e2f_peer_signal")
            for p in peers:
                _lib.check(lib.e2f_peer_wait(may_write(me, p), seq, st), "e2f_peer_wait")
                _lib.check(lib.e2f_peer_copy(self._remote[p][k] + me * nbytes, send.data_ptr(), nbytes, st), "e2f_peer_copy")
                _lib.check(lib.e2f_peer_signal(landed(p, me), seq, st), "e2f_peer_signal")
            _lib.check(lib.e2f_peer_copy(self._local[k] + me * nbytes, send.data_ptr(), nbytes, st), "e2f_peer_copy")
            for p in peers:
                _lib.check(lib.e2f_peer_wait(landed(me, p), seq, st), "e2f_peer_wait")
            done = torch.cuda.Event()
            done.record(side)
        send.record_stream(side)
        return _PendingPeer(done, self._bufs[k], n_valid, send)


def peer_stitch_available(world, device=None):
    """True when the stitch can use peer memory: CUDA, several ranks, all on this node with peer access to this device."""
    if world <= 1 or not torch.cuda.is_available():
        return False
    if int(os.environ.get("LOCAL_WORLD_SIZE", str(world))) != world or torch.cuda.device_count() < world:
        return False
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    return all(r == dev or torch.cuda.can_device_access_peer(dev, r) for r in range(world))


def make_stitcher(num_clips, frames_per_clip, rank, world, payload="fp32", device=None):
    """``PeerStitcher`` on one NVLink box, ``ClipStitcher`` (NCCL / gloo all-gather) otherwise.  The choice is made from
    the same inputs on every rank (world size, ranks on this node, visible devices), so all ranks pick the same class."""
    use_peer = peer_stitch_available(world, device)
    if world > 1 and dist.is_initialized():
        votes = [None] * world
        dist.all_gather_object(votes, bool(use_peer))       # one rank without peer access -> everybody uses the all-gather
        use_peer = all(votes)
    if use_peer:
        return PeerStitcher(num_clips, frames_per_clip, rank, world, payload)
    return ClipStitcher(num_clips, frames_per_clip, rank, world, payload)


def gather_outputs(local_pred, num_clips, frames_per_clip, rank, world, payload="fp32"):
    """Blocking stitch: all-gather per-rank predictions; block sharding means the result is already in clip order.

    local_pred: (share * frames_per_clip, 3, H, W) for this rank's clips, zero-padded to ``padded_share`` clips.
    Returns (num_clips * frames_per_clip, 3, H, W) on every rank."""
    return ClipStitcher(num_clips, frames_per_clip, rank, world, payload).start(local_pred).wait()


@torch.no_grad()
def run_clips(model, clips, num_local_frames, rank=0, world=1, device=None, clips_per_call=8, payload="fp32"):
    """Run ``model`` over this rank's share of ``clips`` (num_clips, T, 3, H, W; same on every rank or only the
    local share is read) and return the stitched (num_clips*T, 3, H, W) predictions on every rank."""
    num_clips, T = clips.shape[0], clips.shape[1]
    mine = shard_clips(num_clips, rank, world)
    share = padded_share(num_clips, world)
    outs = []
    for i in range(0, len(mine), clips_per_call):
        batch = clips[mine[i:i + clips_per_call]]
        if device is not None:
            batch = batch.to(device, non_blocking=True)
        pred, _ = model(batch, num_local_frames)
        outs.append(pred)
    local = torch.cat(outs) if outs else clips.new_zeros((0, 3) + tuple(clips.shape[-2:]))
    if device is not None and local.device != torch.device(device):
        local = local.to(device)
    if local.shape[0] < share * T:
        pad = local.new_zeros((share * T - local.shape[0],) + tuple(local.shape[1:]))
        local = torch.cat([local, pad])
    return gather_outputs(local, num_clips, T, rank, world, payload)
