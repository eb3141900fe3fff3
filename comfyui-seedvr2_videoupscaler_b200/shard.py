"""Clip-parallel sharding across the GPUs of one box (SURVEY.md §8(e)).

The path shards by clip: every rank upscales a contiguous frame range with its own
full copy of the weights (no data-path collective), then ONE all-gather returns the
decoded frames — replacing the reference's mp.Queue + shared-memory + numpy hand-off
(``inference_cli.py:1100, 1227-1232``).  The partition is the reference's:
``total // n`` frames per rank, +1 for the first ``total % n`` ranks, plus
``temporal_overlap`` extra frames on all but the last rank
(``inference_cli.py:1166-1176``; ``partition_preloaded`` is the variant for frames already in memory, ``:1196-1213``).
``stream_shard`` is the same run streamed: each rank streams its range through bounded device memory and only the
frames at the rank seams cross ranks.
"""
from __future__ import annotations

from typing import Iterator, List, Optional, Tuple

import torch


def partition_frames(total: int, n: int, overlap: int = 0, start: int = 0) -> List[Tuple[int, int]]:
    """[start, end) per rank, reference order (inference_cli.py:1166-1193)."""
    base, rem = total // n, total % n
    out, cur = [], start
    for idx in range(n):
        cnt = base + (1 if idx < rem else 0)
        end = cur + cnt
        if idx < n - 1 and overlap > 0:
            end = min(end + overlap, start + total)
        out.append((cur, end))
        cur += cnt
    return out


def partition_preloaded(total: int, n: int, overlap: int = 0, batch_size: int = 1) -> List[Tuple[int, int]]:
    """[start, end) per rank when the whole frame tensor is already in memory (inference_cli.py:1196-1213): without
    overlap ``torch.chunk`` (ceil(total / n) frames per rank, the tail ranks may get fewer or none); with overlap,
    chunks of ``total // n + overlap`` frames rounded up to a multiple of ``batch_size``, stepping by that minus the
    overlap, the last rank running to the end."""
    if overlap > 0 and n > 1:
        cwo = total // n + overlap
        if batch_size > 1:
            cwo = (cwo + batch_size - 1) // batch_size * batch_size
        base = cwo - overlap
        out = []
        for i in range(n):
            s = i * base
            e = total if i == n - 1 else min(s + cwo, total)
            out.append((min(s, total), max(min(s, total), e)))
        return out
    size = -(-total // n)          # torch.chunk
    out, cur = [], 0
    while cur < total:
        out.append((cur, min(cur + size, total)))
        cur += size
    return out


def gather_frames(local: torch.Tensor, counts: List[int], group=None) -> torch.Tensor:
    """All-gather decoded frames (T_r, H, W, C) of every rank into rank order.
    Ranks may hold different frame counts: shards are padded to max(counts) for one
    equal-sized NCCL/gloo all_gather and trimmed afterwards."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    tmax = max(counts)
    T, H, W, C = local.shape
    buf = local
    if T < tmax:
        buf = torch.cat([local, local.new_zeros(tmax - T, H, W, C)], 0)
    out = torch.empty(world, tmax, H, W, C, device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(out.view(-1), buf.reshape(-1).contiguous(), group=group)
    return torch.cat([out[r, :counts[r]] for r in range(world)], 0)


def blend_weights(overlap: int, dtype=torch.bfloat16):
    """Per-frame (w_prev, w_cur) of blend_overlapping_frames (generation_utils.py:299-310), computed with the same
    torch ops in the frames' dtype so that every rounding point matches: Hann cross-fade over the middle third for
    overlap >= 3, linear below."""
    if overlap >= 3:
        t = torch.linspace(0.0, 1.0, steps=overlap, dtype=dtype)
        blend_start, blend_end = 1.0 / 3.0, 2.0 / 3.0
        u = ((t - blend_start) / (blend_end - blend_start)).clamp(0.0, 1.0)
        w_prev = 0.5 + 0.5 * torch.cos(torch.pi * u)
    else:
        w_prev = torch.linspace(1.0, 0.0, steps=overlap, dtype=dtype)
    return w_prev, 1.0 - w_prev


def blend_overlap(prev_tail: torch.Tensor, cur_head: torch.Tensor) -> torch.Tensor:
    """Cross-fade of the ``overlap`` frames two neighbouring ranges share (``blend_overlapping_frames``,
    generation_utils.py:284-312): [overlap, H, W, C] each, bf16 (inside the pipeline) or fp32 (the multi-GPU merge),
    on the GPU (one libsvr2 kernel); weights and rounding points follow the frames' dtype."""
    from . import lib
    assert prev_tail.shape == cur_head.shape and prev_tail.is_cuda
    n = prev_tail.shape[0]
    dt = torch.float32 if prev_tail.dtype == torch.float32 else torch.bfloat16
    a, b = prev_tail.to(dt).contiguous(), cur_head.to(dt).contiguous()
    w_prev, w_cur = blend_weights(n, dt)
    wp, wc = w_prev.float().to(a.device), w_cur.float().to(a.device)
    elems = a[0].numel()
    shape = a.shape
    pad = (-elems) % (4 if dt == torch.float32 else 8)     # the kernels move 16 bytes per thread
    if pad:      # odd frame sizes (e.g. a max_resolution cap that rounds to odd H and W): pad each frame's tail
        a = torch.nn.functional.pad(a.reshape(n, elems), (0, pad))
        b = torch.nn.functional.pad(b.reshape(n, elems), (0, pad))
    out = torch.empty_like(a)
    name = "svr2_blend_overlap_f32" if dt == torch.float32 else "svr2_blend_overlap_bf16"
    lib.call(name, lib.ptr(a), lib.ptr(b), lib.ptr(out), lib.ptr(wp), lib.ptr(wc), n, elems + pad, lib.stream(),
             nbytes=3.0 * a.numel() * a.element_size())
    return out[:, :elems].reshape(shape) if pad else out


def merge_shards(chunks: List[torch.Tensor], overlap: int, blend=None) -> torch.Tensor:
    """Concatenate the per-rank results in rank order, cross-fading the ``overlap`` frames a chunk shares with the
    accumulated result (inference_cli.py:1241-1274; fp32 like the reference).  ``blend(prev_tail, cur_head)``
    defaults to the libsvr2 kernel."""
    blend = blend or blend_overlap
    chunks = [c.float() for c in chunks]
    if overlap <= 0 or len(chunks) == 1:
        return torch.cat(chunks, 0)
    result = chunks[0]
    for c in chunks[1:]:
        if c.shape[0] > overlap and result.shape[0] >= overlap:
            blended = blend(result[-overlap:], c[:overlap])
            result = torch.cat([result[:-overlap], blended, c[overlap:]], 0)
        elif c.shape[0] > overlap:       # chunk too small to blend into: append its non-overlapping part
            result = torch.cat([result, c[overlap:]], 0)
    return result


# ---------------------------------------------------------------------------------------------------------------------
# Streamed multi-GPU runs: every rank streams its own range, only the seam frames cross ranks
# ---------------------------------------------------------------------------------------------------------------------
def blend_seam(prev_tail: torch.Tensor, cur_head: torch.Tensor, f32: bool = True, u8: bool = False):
    """The rank-seam cross-fade of ``stream_shard`` (libsvr2 ``svr2_blend_overlap_u8``, one pass): the fp32 open tail
    [overlap, H, W, C] against the bf16 chunk head of the same shape.  Returns (fp32 frames, exactly those of
    ``blend_overlap(prev_tail, cur_head.float())``, or None when not ``f32``; their CLI bytes, the per-value rule of
    ``color_fix.sample_to_image_u8``, or None when not ``u8``).  Any frame size, no padding copy."""
    from . import lib
    assert prev_tail.shape == cur_head.shape and prev_tail.is_cuda and (f32 or u8)
    assert prev_tail.dtype == torch.float32 and cur_head.dtype == torch.bfloat16
    a, b = prev_tail.contiguous(), cur_head.contiguous()
    n, elems = a.shape[0], a[0].numel()
    w_prev, w_cur = (w.to(a.device) for w in blend_weights(n, torch.float32))
    out_f = torch.empty_like(a) if f32 else None
    out_b = torch.empty(a.shape, dtype=torch.uint8, device=a.device) if u8 else None
    lib.call("svr2_blend_overlap_u8", lib.ptr(a), lib.ptr(b), lib.ptr(out_f), lib.ptr(out_b), lib.ptr(w_prev),
             lib.ptr(w_cur), n, elems, lib.stream(), nbytes=a.numel() * (6.0 + (4.0 if f32 else 0.0) + (1.0 if u8 else 0.0)))
    return out_f, out_b


class MergePlan:
    """What ``merge_shards(chunks, overlap)`` does with chunks of ``lengths`` frames, worked out from the lengths alone
    (every rank computes the same plan without communicating):

    - ``pos[r][i]``: the output position of frame i of chunk r, None when the merge drops it (a chunk no longer than
      ``overlap``, or the head of a chunk when the result is still shorter than ``overlap``);
    - ``blend[r]``: the first position chunk r's head (frames 0 .. overlap-1) is cross-faded into, or None;
    - ``last[j]``: the last chunk that writes position j — its value is final after that chunk's step;
    - ``carry[r]``: the positions some later chunk will still cross-fade, after chunk r's step (the open tail, a suffix
      of the result so far, at most ``overlap`` frames);
    - ``length``: the frame count of the merged result."""

    def __init__(self, lengths: List[int], overlap: int):
        n = len(lengths)
        blending = overlap > 0 and n > 1
        self.pos, self.blend, length = [], [], 0
        for r, L in enumerate(lengths):
            if not blending or r == 0:
                self.pos.append(list(range(length, length + L)))
                self.blend.append(None)
                length += L
            elif L > overlap and length >= overlap:
                self.blend.append(length - overlap)
                self.pos.append(list(range(length - overlap, length)) + list(range(length, length + L - overlap)))
                length += L - overlap
            else:
                self.blend.append(None)
                self.pos.append([None] * overlap + list(range(length, length + L - overlap)) if L > overlap
                                else [None] * L)
                length += max(0, L - overlap)
        self.length = length
        self.last = [0] * length
        ends = []
        for r, ps in enumerate(self.pos):
            for j in ps:
                if j is not None:
                    self.last[j] = r
            ends.append(max([j + 1 for j in ps if j is not None], default=ends[-1] if ends else 0))
        self.carry = [[j for j in range(max(0, e - overlap), e) if self.last[j] > r] for r, e in enumerate(ends)]


def _peer(t: torch.Tensor, peer: int, group, device, send: bool) -> Optional[torch.Tensor]:
    """Send ``t`` (fp32 frames) to, or receive it from, rank ``peer`` of ``group``: its shape first, then the frames;
    on the device with NCCL, staged through host memory otherwise (gloo)."""
    import torch.distributed as dist
    on_dev = dist.get_backend(group) == "nccl"
    where = device if on_dev else torch.device("cpu")
    if send:
        dist.send(torch.tensor(t.shape, dtype=torch.int64, device=where), group=group, group_dst=peer)
        dist.send(t.to(where).contiguous(), group=group, group_dst=peer)
        return None
    shape = torch.empty(4, dtype=torch.int64, device=where)
    dist.recv(shape, group=group, group_src=peer)
    out = torch.empty(shape.tolist(), dtype=torch.float32, device=where)
    dist.recv(out, group=group, group_src=peer)
    return out.to(device)


_OUT, _KEEP, _SKIP = 0, 1, 2      # frame kinds of one rank: formatted and yielded, kept on the device for a seam, neither


def stream_shard(engine, frames, *, group=None, total: Optional[int] = None,
                 ranges: Optional[List[Tuple[int, int]]] = None, out_dtype: torch.dtype = torch.uint8,
                 **options) -> Iterator[Tuple[int, torch.Tensor]]:
    """One video over the ranks of ``group`` (torch.distributed; None: the default group), each streaming its own frame
    range through bounded device memory: the streamed form of ``partition_frames`` + per-rank ``upscale_video`` +
    ``merge_shards`` + the prepend drop, the reference CLI's multi-GPU run (inference_cli.py:1127-1288).  Every rank
    calls it with the same arguments and its own engine.

    ``frames``: the whole video as one host tensor (T,h,w,C), or a callable ``open(start, end)`` returning source frames
    [start, end) as a tensor or an iterable of chunks (a decoder seeking to its range); ``total`` (the frame count) is
    then required.  ``options``: those of ``upscale_video`` (``temporal_overlap``, ``prepend_frames``, the tiling
    settings, …), applied to every rank's batch loop as they are: every rank seeds alike and starts its own
    input-noise generator.  ``prepend_frames`` = p puts the p mirrored frames in front of the video once; the video
    then has ``total + p`` frames.  ``ranges``: [start, end) per rank in those frames (``partition_preloaded(...)``,
    say), default ``partition_frames(total + p, world, temporal_overlap)``; ranks past the end of a shorter list get
    no frames.

    Yields ``(global_index, frames)``: this rank's share of the result, each (t,H,W,C) in pinned host memory, as soon
    as nothing can change it — the frames no seam touches as their batches finish, in order, then the seam frames the
    cross-fade with the previous ranks made final (they precede those).  An image-sequence writer writes each frame
    under its index; the shares of the ranks are consecutive index ranges in rank order.  ``out_dtype``:
    ``torch.uint8`` (the CLI's 8-bit frames: ``(merged * 255)`` truncated) or ``torch.float32`` (the merged frames);
    not bf16, as the cross-faded seam frames are fp32 values.

    When its batch loop has ended, a rank receives the open tail of the result (fp32, at most ``temporal_overlap``
    frames) from the previous rank, cross-fades its head into it (``blend_seam``), yields what became final and sends
    the new open tail on; a rank whose chunk the merge skips forwards it.  Nothing else crosses ranks.  Device memory:
    that of ``stream_video`` plus at most 2 * ``temporal_overlap`` frames (the head waiting for the tail, and the
    rank's own tail).  Every rank must run its generator to the end: a consumer that stops early leaves the later
    ranks waiting for the tail."""
    import inspect

    import torch.distributed as dist

    from . import pipeline
    if out_dtype not in (torch.uint8, torch.float32):
        raise ValueError(f"out_dtype must be torch.uint8 or torch.float32, got {out_dtype}")
    args = inspect.signature(pipeline.SeedVR2Engine.upscale_video).bind(engine, None, **options)
    args.apply_defaults()
    opt = dict(args.arguments)
    tiling = pipeline.tiling_settings(opt.pop("tiling"))
    p, overlap = opt["prepend_frames"], opt["temporal_overlap"]
    if p < 0:
        raise ValueError(f"prepend_frames must be >= 0, got {p}")
    if isinstance(frames, torch.Tensor):
        if total is not None and total != frames.shape[0]:
            raise ValueError(f"total={total} but the video has {frames.shape[0]} frames")
        total, video = frames.shape[0], frames
        read = lambda s, e: video[s:e]
    elif callable(frames):
        if total is None:
            raise ValueError("a frame reader open(start, end) needs total, the video's frame count")
        read = frames
    else:
        raise TypeError("frames must be a tensor or a callable open(start, end)")
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = total + p if total > 0 else 0
    if ranges is None:
        ranges = partition_frames(n, world, overlap)
    ranges = [(int(a), int(b)) for a, b in ranges]
    if len(ranges) > world:
        raise ValueError(f"{len(ranges)} ranges for {world} ranks")
    ranges += [(n, n)] * (world - len(ranges))
    for r, (a, b) in enumerate(ranges):
        if not 0 <= a <= b <= n or (r > 0 and not ranges[r - 1][0] <= a <= ranges[r - 1][1]) or (r == 0 and a != 0):
            raise ValueError(f"ranges must run from 0 to {n} in order without gaps, got {ranges}")
    if ranges[-1][1] != n:
        raise ValueError(f"ranges must end at frame {n} (total + prepend_frames), got {ranges}")
    return _stream_ranks(engine, read, total, ranges, rank, group, out_dtype, opt, tiling) if n else iter(())


def _stream_ranks(engine, read, total, ranges, rank, group, out_dtype, opt, tiling):
    """The body of ``stream_shard`` once its arguments are checked."""
    from . import pipeline
    world, p, overlap = len(ranges), opt["prepend_frames"], opt["temporal_overlap"]
    blending = overlap > 0 and world > 1
    plan = MergePlan([b - a for a, b in ranges], overlap if blending else 0)
    drop = p if 0 < p < plan.length else 0
    pos = plan.pos[rank]
    kind = [_SKIP if j is None else
            _KEEP if plan.last[j] > rank or (plan.blend[rank] is not None and i < overlap) else
            _OUT if j >= drop else _SKIP for i, j in enumerate(pos)]
    cuda = engine.device.type == "cuda"
    f32 = out_dtype == torch.float32

    def to_host(t):
        h = torch.empty(t.shape, dtype=t.dtype, pin_memory=cuda)
        h.copy_(t, non_blocking=cuda)
        return h

    posted = [0]

    def finish(sample, style, src):
        """Phase 4 once per slice, then each run of frames of one kind formatted as that kind needs."""
        lo = posted[0]
        posted[0] += sample.shape[0]
        sample, image = engine.correct_clip(sample, style, src, opt["color_correction"])
        pieces, i = [], lo
        while i < posted[0]:
            k = i
            while k < posted[0] and kind[k] == kind[i] and (kind[i] != _OUT or pos[k] - pos[i] == k - i):
                k += 1
            s_, im = sample[i - lo:k - lo], None if image is None else image[i - lo:k - lo]
            if kind[i] == _KEEP:           # bf16 images that own their memory
                pieces.append((_KEEP, i, engine.format_image(s_, None if im is None else im.clone())))
            elif kind[i] == _OUT:
                img = engine.format_image(s_, im, torch.bfloat16 if f32 else torch.uint8)
                pieces.append((_OUT, i, img.float() if f32 else img))
            i = k
        return pieces

    kept = {}                       # local frame -> bf16 image (1,H,W,C) on the device, until the seam step

    def stage(done):
        host = []
        for pieces in done:
            for what, i, t in pieces:
                if what == _KEEP:
                    for d in range(t.shape[0]):
                        kept[i + d] = t[d:d + 1]
                else:
                    host.append((pos[i] - drop, to_host(t)))
        ev = None
        if cuda and host:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(engine.device))
        return host, ev

    a, b = ranges[rank]
    if b > a:
        src = pipeline.RangeSource(read, total, a, b, prepend=p)
        prev = None
        for done in engine._final_slices(src, opt["batch_size"], overlap, opt["seed"], opt["color_correction"],
                                         opt["resolution"], opt["max_resolution"], opt["keep_alpha"],
                                         opt["input_noise_scale"], opt["latent_noise_scale"],
                                         opt["uniform_batch_size"], 0, tiling=tiling, finish=finish):
            cur = stage(done)
            del done
            if prev is not None:
                if prev[1] is not None:
                    prev[1].synchronize()
                yield from prev[0]
            prev = cur
        if prev is not None:
            if prev[1] is not None:
                prev[1].synchronize()
            yield from prev[0]
    if not blending:
        return

    # the seam step: take the open tail from the previous rank, cross-fade, yield what became final, pass the tail on
    tail_pos = plan.carry[rank - 1] if rank > 0 else []
    tail = _peer(None, rank - 1, group, engine.device, send=False) if tail_pos else None
    if tail is not None and tail.shape[0] != len(tail_pos):
        raise RuntimeError(f"rank {rank}: received an open tail of {tail.shape[0]} frames, expected {len(tail_pos)}")
    open_tail = [] if tail is None else [(j, tail[k:k + 1]) for k, j in enumerate(tail_pos)]
    w0, seam = plan.blend[rank], None
    if w0 is not None:
        final = sum(1 for j in range(w0, w0 + overlap) if plan.last[j] == rank)      # a prefix of the window
        head = torch.cat([kept.pop(i) for i in range(overlap)], 0)
        out_f, out_b = blend_seam(tail, head, f32=f32 or final < overlap, u8=not f32 and final > 0)
        skip = max(0, drop - w0)                    # window frames before the prepend drop are not yielded
        if final > skip:
            seam = (w0 + skip - drop, to_host((out_f if f32 else out_b)[skip:final]))
        open_tail = [(w0 + k, out_f[k:k + 1]) for k in range(final, overlap)]
    open_tail += [(pos[i], kept.pop(i).float()) for i in sorted(kept)]
    assert [j for j, _ in open_tail] == plan.carry[rank], (rank, [j for j, _ in open_tail], plan.carry[rank])
    if rank < world - 1 and plan.carry[rank]:       # the next ranks wait for this, not for the consumer
        _peer(torch.cat([t for _, t in open_tail], 0), rank + 1, group, engine.device, send=True)
    if seam is not None:
        if cuda:
            torch.cuda.current_stream(engine.device).synchronize()
        yield seam
