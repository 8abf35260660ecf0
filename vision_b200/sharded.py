"""Multi-GPU: the hot path shards on the batch / image dimension (SURVEY.md §8e).

One process per GPU (torchrun), each rank runs the op on its own images, and the per-shard outputs are exchanged with
an all-gather over NCCL (NVLink 5 / NVSwitch) - no reduce, no all-to-all, nothing else.

* ``all_gather_equal``  - one ``all_gather_into_tensor`` of equal-shaped outputs.
* ``sharded_apply_overlapped`` - the same exchange hidden behind the compute: the shard is cut into chunks along dim 0,
  chunk i is computed on the compute stream and its all-gather is issued on a side stream as soon as the chunk is
  ready, so chunk i's transfer runs under chunk i+1's kernel (NVSwitch gives every GPU full bandwidth to every peer,
  so the gather of a chunk costs about (world-1)/world * bytes / 0.9 TB/s and is hidden when the kernel takes longer).
  The gathered result is returned as a VIEW ``[world * n, ...]`` over a ``[chunks, world, chunk, ...]`` buffer (no
  re-packing pass).
* NMS keep-lists (data-dependent length) travel padded, with their length in front, so each image is one fixed-size
  message; ``sharded_batched_nms`` runs all local images without a host synchronisation and gathers once.

The helpers are backend-agnostic (nccl on GPUs; gloo in the CPU tests of the plumbing).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch
import torch.distributed as dist


def shard_bounds(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced split of n units: the first (n % world) ranks get one extra."""
    base, rem = divmod(n, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def _world(group=None) -> tuple[int, int]:
    if not dist.is_available() or not dist.is_initialized():
        return 0, 1
    return dist.get_rank(group), dist.get_world_size(group)


def _gather_into(out: torch.Tensor, local: torch.Tensor, group=None) -> None:
    """out [world, *local.shape] <- every rank's `local` (one collective)."""
    world = out.shape[0]
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(out, local, group=group)
    else:
        dist.all_gather(list(out.unbind(0)), local, group=group)


def all_gather_equal(local: torch.Tensor, group=None) -> torch.Tensor:
    """All ranks hold the same shape: returns cat over ranks along dim 0 (one collective)."""
    rank, world = _world(group)
    if world == 1:
        return local
    local = local.contiguous()
    out = torch.empty((world,) + tuple(local.shape), dtype=local.dtype, device=local.device)
    _gather_into(out, local, group)
    return out.reshape((world * local.shape[0],) + tuple(local.shape[1:]))


def all_gather_varlen(local: torch.Tensor, capacity: int, group=None) -> list[torch.Tensor]:
    """1-D int64 lists of data-dependent length <= capacity: one padded all-gather.
    Returns the per-rank lists (rank order)."""
    rank, world = _world(group)
    assert local.dim() == 1 and local.dtype == torch.int64 and local.numel() <= capacity
    if world == 1:
        return [local]
    buf = torch.full((capacity + 1,), -1, dtype=torch.int64, device=local.device)
    buf[0] = local.numel()
    buf[1:1 + local.numel()] = local
    gathered = all_gather_equal(buf.unsqueeze(0), group=group)      # [world, capacity + 1]
    lens = gathered[:, 0].tolist()
    return [gathered[r, 1:1 + int(lens[r])] for r in range(world)]


def sharded_apply(fn: Callable[..., torch.Tensor], local_inputs: Sequence, group=None) -> torch.Tensor:
    """Run `fn(*local_inputs)` on this rank's shard and all-gather the equal-shaped outputs."""
    return all_gather_equal(fn(*local_inputs), group=group)


class OverlappedGather:
    """Chunked all-gather on a side stream (see module docstring).  Reusable: buffers and the side stream persist."""

    def __init__(self, group=None):
        self.group = group
        self.rank, self.world = _world(group)
        self._stream: Optional[torch.cuda.Stream] = None
        self._buf: Optional[torch.Tensor] = None

    def _side(self, device) -> Optional["torch.cuda.Stream"]:
        if device.type != "cuda":
            return None
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=device)
        return self._stream

    def run(self, chunk_fn: Callable[[int], torch.Tensor], chunks: int) -> torch.Tensor:
        """chunk_fn(i) -> this rank's output for chunk i (all chunks and all ranks: same shape).  Returns the gathered
        result as a [world * chunks * m, ...] view in rank-major order (rank r's rows are contiguous in the view)."""
        world = self.world
        if world == 1:
            outs = [chunk_fn(i) for i in range(chunks)]
            return outs[0] if chunks == 1 else torch.cat(outs, dim=0)
        first = chunk_fn(0)
        dev = first.device
        shape = (chunks, world) + tuple(first.shape)
        if self._buf is None or tuple(self._buf.shape) != shape or self._buf.dtype != first.dtype or self._buf.device != dev:
            self._buf = torch.empty(shape, dtype=first.dtype, device=dev)
        buf = self._buf
        side = self._side(dev)
        cur = first
        for i in range(chunks):
            local = cur.contiguous()
            if side is not None:
                ready = torch.cuda.Event()
                ready.record(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):
                    side.wait_event(ready)
                    local.record_stream(side)
                    _gather_into(buf[i], local, self.group)
            else:
                _gather_into(buf[i], local, self.group)
            if i + 1 < chunks:
                cur = chunk_fn(i + 1)          # runs on the compute stream while chunk i travels
        if side is not None:
            torch.cuda.current_stream(dev).wait_stream(side)
        return _rank_major_view(buf)


def _rank_major_view(buf: torch.Tensor) -> torch.Tensor:
    """[chunks, world, m, ...] -> rank-major [world, chunks * m, ...] without copying when chunks == 1; otherwise a
    permuted (non-contiguous) view that indexes like the concatenation over ranks of each rank's chunks in order."""
    chunks, world, m = buf.shape[:3]
    v = buf.transpose(0, 1)                                  # [world, chunks, m, ...], strided
    return v.reshape((world * chunks * m,) + tuple(buf.shape[3:])) if chunks == 1 else _LazyCat(v)


class _LazyCat:
    """Rank-major result of a chunked gather: behaves like the [world * chunks * m, ...] tensor for the common
    consumers (``shape``, ``__getitem__`` of a rank slice, ``contiguous()``, ``materialize()``) without paying the
    re-packing pass unless the caller asks for one contiguous tensor."""

    def __init__(self, v: torch.Tensor):
        self.v = v                                            # [world, chunks, m, ...]
        w, c, m = v.shape[:3]
        self.shape = torch.Size((w * c * m,) + tuple(v.shape[3:]))
        self.dtype, self.device = v.dtype, v.device

    def rank(self, r: int) -> torch.Tensor:
        """Rank r's output as a [chunks, m, ...] view (each chunk contiguous)."""
        return self.v[r]

    def materialize(self) -> torch.Tensor:
        return self.v.reshape(self.shape)                     # one packing copy

    contiguous = materialize

    def __len__(self) -> int:
        return self.shape[0]


def sharded_apply_overlapped(fn: Callable[[torch.Tensor], torch.Tensor], local: torch.Tensor, chunks: int = 4,
                             gather: Optional[OverlappedGather] = None, group=None):
    """fn over `local` (split along dim 0 into `chunks` equal parts) with the all-gather of each part's output hidden
    behind the next part's kernel.  Returns a tensor (world == 1 or chunks == 1) or a `_LazyCat` rank-major view."""
    n = local.shape[0]
    chunks = max(1, min(chunks, n))
    while n % chunks:
        chunks -= 1
    step = n // chunks
    g = gather or OverlappedGather(group)
    return g.run(lambda i: fn(local[i * step:(i + 1) * step]), chunks)


def sharded_batched_nms(fn: Callable[..., torch.Tensor], problems: Sequence[tuple], iou_threshold: float,
                        capacity: Optional[int] = None, group=None) -> list[list[torch.Tensor]]:
    """`problems` = this rank's images, each (boxes, scores, idxs).  A single image's NMS is never split
    (greedy dependency); images are the shard unit.  Returns keep lists for every rank's images.
    `capacity` = static upper bound, IDENTICAL on every rank, of (boxes + images) per rank; defaults to
    this rank's own total, which is only valid when all ranks hold equally many boxes (weak scaling)."""
    rank, world = _world(group)
    keeps = [fn(b, s, i, iou_threshold) for (b, s, i) in problems]
    if world == 1:
        return [keeps]
    cap = capacity if capacity is not None else sum(int(b.shape[0]) + 1 for (b, _, _) in problems)
    device = problems[0][0].device if problems else torch.device("cpu")
    packed = torch.cat([torch.cat([torch.tensor([k.numel()], dtype=torch.int64, device=device), k]) for k in keeps]) \
        if keeps else torch.empty(0, dtype=torch.int64, device=device)
    per_rank = all_gather_varlen(packed, cap, group=group)
    out = []
    for flat in per_rank:
        lst, pos = [], 0
        while pos < flat.numel():
            n = int(flat[pos])
            lst.append(flat[pos + 1:pos + 1 + n])
            pos += 1 + n
        out.append(lst)
    return out


def sharded_batched_nms_padded(problems: Sequence[tuple], iou_threshold: float, group=None) -> tuple[torch.Tensor, torch.Tensor]:
    """Device-resident variant for equally sized images (n boxes each): runs ``vision_b200::batched_nms_padded`` on every
    local image WITHOUT a host synchronisation, then ONE all-gather of the padded keep lists (count in front of each).
    Returns (keep [world, images, n] int64, count [world, images] int64); keep[r, j, :count[r, j]] are image j of rank r's
    kept indices in descending-score order."""
    from . import _lib

    _lib.load_ops()
    rank, world = _world(group)
    keeps, counts = [], []
    for (b, s, i) in problems:
        k, c = torch.ops.vision_b200.batched_nms_padded(b, s, i, float(iou_threshold))
        keeps.append(k)
        counts.append(c)
    keep = torch.stack(keeps)                                  # [images, n]
    count = torch.cat(counts)                                  # [images]
    if world == 1:
        return keep.unsqueeze(0), count.unsqueeze(0)
    packed = torch.cat([count.unsqueeze(1), keep], dim=1)      # [images, 1 + n]: one fixed-size message per image
    g = torch.empty((world,) + tuple(packed.shape), dtype=packed.dtype, device=packed.device)
    _gather_into(g, packed, group)
    return g[:, :, 1:], g[:, :, 0]


# ---- all-gather fused into the producing kernel (peer stores over NVLink / NVSwitch) -------------------------------------
class PeerGather:
    """Gathered output buffers ``[2, world, *shard_shape]`` in symmetric (peer-mapped) device memory.

    With it the all-gather that follows a sharded op is not a collective call at all: the op's kernel stores every
    finished output element to its own slot in ALL ranks' buffers (``dst_ptrs``: the local slot first, then the same
    slot of each peer, mapped through ``torch.distributed._symmetric_memory``), so the exchange travels over NVLink
    while the kernel is still streaming its input from HBM - for resize the output is 0.6 % of the input bytes.
    ``barrier()`` is a stream-ordered device-side barrier over the ranks (no host sync), issued ONCE per step, after the
    kernel: every peer's stores have landed.  Steps alternate between the two buffers, so the rewrite of a buffer two
    steps later is already ordered behind every rank's reads of it (each rank passes the barrier of the step in between
    only after all ranks reached it, i.e. after their stream-ordered consumers of the older buffer).

    ``PeerGather.create`` returns None where peer mapping is not available (CPU / gloo, one rank, driver without
    fabric or fd handle export); callers then use the NCCL exchange (`sharded_apply_overlapped`)."""

    def __init__(self, buf: torch.Tensor, hdl, rank: int, world: int):
        self.buf, self.hdl, self.rank, self.world = buf, hdl, rank, world          # buf: [2, world, *shard]
        shard_bytes = buf[0, 0].numel() * buf.element_size()
        half = world * shard_bytes
        order = [rank] + [r for r in range(world) if r != rank]
        self._dst = [[int(hdl.buffer_ptrs[r]) + k * half + rank * shard_bytes for r in order] for k in range(2)]
        # NVSwitch multicast address of this rank's slot (0 when the box / allocation has no multicast object): ONE store to
        # it is replicated by the switch into every rank's buffer (multimem.st), instead of world - 1 peer stores
        mc = 0
        try:
            mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
        except Exception:                            # noqa: BLE001
            mc = 0
        self._mc = [mc + k * half + rank * shard_bytes if mc else 0 for k in range(2)]
        self.cur = 1

    @classmethod
    def create(cls, shard_shape: Sequence[int], dtype: torch.dtype, device, group=None) -> Optional["PeerGather"]:
        rank, world = _world(group)
        if world < 2 or world > 8 or torch.device(device).type != "cuda" or dist.get_backend(group) != "nccl":
            return None
        try:
            import torch.distributed._symmetric_memory as symm

            buf = symm.empty((2, world) + tuple(shard_shape), dtype=dtype, device=device)
            hdl = symm.rendezvous(buf, group if group is not None else dist.group.WORLD)
            if len(hdl.buffer_ptrs) != world:
                return None
            return cls(buf, hdl, rank, world)
        except Exception as e:                       # noqa: BLE001 - any failure of the optional transport means "use NCCL"
            import warnings

            warnings.warn(f"vision_b200.sharded.PeerGather: symmetric memory unavailable ({type(e).__name__}: {e}); using NCCL")
            return None

    @property
    def shard_shape(self):
        return tuple(self.buf.shape[2:])

    def advance(self) -> None:
        """Switch to the other buffer (call once per step, before the op)."""
        self.cur ^= 1

    @property
    def dst_ptrs(self):
        return self._dst[self.cur]

    @property
    def mc_ptr(self) -> int:
        return self._mc[self.cur]

    def barrier(self) -> None:
        self.hdl.barrier(channel=0)

    def gathered(self) -> torch.Tensor:
        """Rank-major ``[world * n, ...]`` view of the current buffer."""
        b = self.buf[self.cur]
        return b.reshape((b.shape[0] * b.shape[1],) + tuple(b.shape[2:]))


def resize_gather(local: torch.Tensor, size, peer: Optional[PeerGather], interpolation="bilinear", antialias: bool = True,
                  group=None):
    """``resize(local, size)`` on this rank's images + all-gather of the outputs over the ranks, rank-major.

    With a `PeerGather` buffer the exchange is fused into the resize kernel (peer stores); otherwise the NCCL exchange
    chunked under the kernel (`sharded_apply_overlapped`).  ``local`` is ``[n, C, H, W]``; size is ``[h, w]``."""
    from . import _lib, transforms

    rank, world = _world(group)
    if peer is None or world == 1:
        return sharded_apply_overlapped(lambda t: transforms.resize_image(t, size, interpolation=interpolation, antialias=antialias),
                                        local, chunks=4, group=group)
    n, c, ih, iw = local.shape
    oh, ow = transforms.compute_resized_output_size((ih, iw), size=size)
    assert peer.shard_shape == (n, c, oh, ow) and peer.buf.dtype == local.dtype, "PeerGather buffer does not match the output shard"
    _lib.load_ops()
    mode = transforms._MODE_CODE[transforms._mode_value(interpolation)]
    peer.advance()
    torch.ops.vision_b200.resize_gather(local, peer.dst_ptrs, oh, ow, mode, bool(antialias))
    peer.barrier()                                   # every rank's stores have landed everywhere
    return peer.gathered()


def roi_align_gather(input: torch.Tensor, rois: torch.Tensor, peer: Optional[PeerGather], output_size=(7, 7), spatial_scale: float = 1.0,
                     sampling_ratio: int = -1, aligned: bool = False, multicast: bool = True, group=None):
    """``roi_align`` of this rank's RoIs + all-gather of the ``[K, C, PH, PW]`` outputs over the ranks, rank-major.

    With a `PeerGather` buffer the exchange is fused into the kernel: every finished bin is stored to all ranks' buffers - one
    NVSwitch multicast store (``multimem.st``) when the buffer has a multicast address and ``multicast`` is set, otherwise one
    NVLink peer store per rank.  Without a buffer: the op followed by one NCCL all-gather."""
    from . import _lib, ops as _ops

    rank, world = _world(group)
    ph, pw = (output_size, output_size) if isinstance(output_size, int) else tuple(output_size)
    if peer is None or world == 1:
        return all_gather_equal(_ops.roi_align(input, rois, (ph, pw), spatial_scale, sampling_ratio, aligned), group=group)
    k, c = rois.shape[0], input.shape[1]
    assert peer.shard_shape == (k, c, ph, pw) and peer.buf.dtype == input.dtype, "PeerGather buffer does not match the output shard"
    _lib.load_ops()
    peer.advance()
    mc = peer.mc_ptr if (multicast and input.dtype == torch.float32) else 0
    torch.ops.vision_b200.roi_align_gather(input, rois, peer.dst_ptrs, mc, float(spatial_scale), ph, pw, int(sampling_ratio), bool(aligned))
    peer.barrier()
    return peer.gathered()


def deform_conv2d_gather(input: torch.Tensor, offset: torch.Tensor, weight: torch.Tensor, bias, peer: Optional[PeerGather],
                         stride=(1, 1), padding=(0, 0), dilation=(1, 1), mask=None, group=None):
    """``deform_conv2d`` on this rank's images + all-gather of the ``[n, C_out, H, W]`` outputs over the ranks, rank-major.

    With a `PeerGather` buffer the wgmma kernel's epilogue stores every output element to all ranks' buffers (NVLink peer
    stores); without one: the op followed by the NCCL exchange."""
    from . import _lib, ops as _ops

    rank, world = _world(group)
    if peer is None or world == 1:
        return all_gather_equal(_ops.deform_conv2d(input, offset, weight, bias, stride, padding, dilation, mask), group=group)
    use_mask = mask is not None
    if mask is None:
        mask = torch.zeros((input.shape[0], 1), device=input.device, dtype=input.dtype)
    if bias is None:
        bias = torch.zeros(weight.shape[0], device=input.device, dtype=input.dtype)
    (sh, sw), (ph, pw), (dh, dw) = _ops._pair(stride), _ops._pair(padding), _ops._pair(dilation)
    kh, kw = weight.shape[-2:]
    n_offset_grps = offset.shape[1] // (2 * kh * kw)
    n_weight_grps = input.shape[1] // weight.shape[1]
    assert peer.shard_shape == (input.shape[0], weight.shape[0]) + tuple(offset.shape[2:]) and peer.buf.dtype == input.dtype, \
        "PeerGather buffer does not match the output shard"
    _lib.load_ops()
    peer.advance()
    torch.ops.vision_b200.deform_conv2d_gather(input, weight, offset, mask, bias, peer.dst_ptrs, sh, sw, ph, pw, dh, dw, n_weight_grps,
                                               n_offset_grps, use_mask)
    peer.barrier()
    return peer.gathered()
