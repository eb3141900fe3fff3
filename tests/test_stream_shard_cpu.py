"""CPU, gloo, world sizes 2 and 3: shard.stream_shard with the engine's GPU stages stubbed (as in test_stream_cpu.py)
and its seam kernel restated in torch, against the multi-GPU contract it streams — per-rank upscale_video on the
ranges of the video with the mirrored frames in front, merge_shards, the prepend drop — over a grid of lengths,
overlaps, batch sizes, prepend counts, both partitions and both kinds of source, in float32 and uint8."""
import importlib
import itertools
import os
import sys
import weakref

import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "comfyui_seedvr2_videoupscaler_b200."


def mod(m):
    return importlib.import_module(NAME + m)


def u8_rule(v):
    """svr2_sample_to_image_u8's byte of an fp32 value: * 255, truncated, saturating, NaN -> 0."""
    return torch.nan_to_num(v * 255.0, nan=0.0).clamp(0, 255).to(torch.uint8)


def seam_restated(prev, cur, f32=True, u8=False):
    """svr2_blend_overlap_u8 in torch: three separately rounded fp32 ops, then the byte rule."""
    wp, wc = (w.view(-1, 1, 1, 1) for w in mod("shard").blend_weights(prev.shape[0], torch.float32))
    v = prev * wp + cur.float() * wc
    return (v if f32 else None), (u8_rule(v) if u8 else None)


class Live:
    """Frames of the bf16 images made by the formatting stand-ins that are still alive."""

    def __init__(self):
        self.refs = []

    def add(self, t):
        self.refs.append(weakref.ref(t))
        return t

    def frames(self):
        return sum(r().shape[0] for r in self.refs if r() is not None)


def stub_engine(set_=setattr, live=None):
    """test_stream_cpu.py's stand-ins, set with ``set_`` (plain setattr in a worker process, which is thrown away
    afterwards; monkeypatch.setattr in the test's own process)."""
    pipeline, preprocess, color_fix, alpha, shard, gen_noise = (
        mod(m) for m in ("pipeline", "preprocess", "color_fix", "alpha", "shard", "noise"))
    from oracle import noise_oracle as no
    eng = object.__new__(pipeline.SeedVR2Engine)
    eng.device = torch.device("cpu")

    def fake_run(self, x, channels_last):
        (H, W), _ = preprocess.resized_size(x.shape[1], x.shape[2], self.resolution, self.max_resolution)
        y = torch.nn.functional.interpolate(x[..., :3].permute(0, 3, 1, 2).float(), size=(H, W)).permute(1, 0, 2, 3)
        y = torch.nn.functional.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16))
        return (y * 2 - 1).to(torch.bfloat16).contiguous()

    def fake_alpha(src, sample, image):
        image[..., 3] = src[..., 3].float().mean(dim=(1, 2)).view(-1, 1, 1).to(image.dtype)
        return image

    keep = (lambda t: t) if live is None else live.add
    to_image = lambda s_: keep((s_.float().permute(0, 2, 3, 1).clamp(-1, 1) * 0.5 + 0.5).to(torch.bfloat16))

    def fake_rgba(sample, image):
        image[..., :3] = to_image(sample)
        return keep(image)

    def fake_u8(sample, image_rgba=None):
        img = to_image(sample) if image_rgba is None else fake_rgba(sample, image_rgba.clone())
        return (img.float() * 255.0).to(torch.uint8)

    set_(preprocess.VideoTransform, "run", fake_run)
    set_(gen_noise, "add_input_noise", lambda x, n, scale: no.input_noise(x, n, scale).contiguous())
    eng.vae_encode = lambda x: x[0, ::4, ::8, ::8, None].expand(-1, -1, -1, 16).contiguous()
    eng.inference = lambda noise, latent, **kw: latent + noise * 0.01
    eng.clip_workspace = lambda T, Hp, Wp: None
    eng.vae_decode = lambda z: z[..., 0].repeat_interleave(4, 0)[: 4 * z.shape[0] - 3, None].expand(-1, 3, -1, -1) \
        .repeat_interleave(8, -2).repeat_interleave(8, -1).permute(1, 0, 2, 3).contiguous()
    set_(color_fix, "apply_color_correction",
         lambda s_, st, mode, debug=None: ((s_.float() + st.float()) / 2).to(torch.bfloat16))
    set_(color_fix, "sample_to_image", to_image)
    set_(color_fix, "sample_to_image_rgba", fake_rgba)
    set_(color_fix, "sample_to_image_u8", fake_u8)
    set_(alpha, "upscale_into_image", fake_alpha)
    set_(shard, "blend_overlap", lambda p, c: ((p.float() + c.float()) / 2).to(p.dtype))
    set_(shard, "blend_seam", seam_restated)
    return eng


def video(total, channels=3):
    g = torch.Generator().manual_seed(total * 7 + channels)
    v = torch.rand(total, 16, 24, channels, generator=g)
    if channels == 4:
        v[..., 3] = (torch.arange(total).float() / 16).view(total, 1, 1)
    return v


def odd_chunks(t, seed):
    """An iterable over t in chunks of 1 to 4 frames (empty ones between)."""
    g = torch.Generator().manual_seed(seed)
    pos = 0
    while pos < t.shape[0]:
        k = int(torch.randint(0, 5, (1,), generator=g))
        yield t[pos:pos + k]
        pos += k


def grid(world):
    """(ranges kind, total, overlap, batch, p, source, out dtype, options) covering empty ranks, chunks no longer than
    the overlap, a first chunk shorter than it, cascading seams, p beyond rank 0's share and p beyond the output."""
    cases = []
    for total, ov, bs, p in itertools.product((1, 2, 4, 7, 11, 16), (0, 1, 2, 3, 4), (1, 3, 5), (0, 2, 6, 20)):
        if (total + ov + bs + p) % 3 != world % 3 and not (total <= world or ov >= 3):
            continue                                             # thin the grid; keep all short and deep-overlap cases
        for part in ("frames", "preloaded"):
            i = len(cases)
            cases.append(dict(part=part, total=total, overlap=ov, batch_size=bs, p=p,
                              source="open" if i % 2 else "tensor", out="u8" if i % 3 else "f32",
                              kw=dict(seed=5, resolution=16, keep_alpha=(i % 5 == 0), uniform_batch_size=(i % 7 == 0),
                                      color_correction="lab" if i % 4 == 0 else "none")))
    # seams that cascade through chunks shorter than 2 * overlap (three ranks), and explicit ranges whose last chunk
    # the merge skips, so that the output is shorter than the video: p reaches past it (all frames kept) or not
    extra = [dict(part="preloaded", total=t, overlap=o, batch_size=bs, p=p)
             for t, o, bs, p in ((1, 2, 1, 4), (1, 3, 1, 7), (2, 2, 3, 3), (3, 2, 2, 5), (4, 3, 5, 6))] if world == 3 else []
    extra += [dict(part="custom", total=2, overlap=3, batch_size=2, p=3, ranges=[(0, 2), (2, 5)]),
              dict(part="custom", total=4, overlap=2, batch_size=3, p=1, ranges=[(0, 3), (3, 5)]),
              dict(part="custom", total=3, overlap=1, batch_size=1, p=4, ranges=[(0, 4), (3, 7)])]
    for c in extra:
        for source, out in (("open", "u8"), ("tensor", "f32")):
            i = len(cases)
            cases.append(dict(c, source=source, out=out, kw=dict(seed=5, resolution=16, keep_alpha=(i % 3 == 0),
                                                                 color_correction="lab")))
    return cases


def ranges_for(case, world):
    shard = mod("shard")
    n = case["total"] + case["p"]
    if case["part"] == "custom":
        return case["ranges"], case["ranges"] + [(n, n)] * (world - len(case["ranges"]))
    if case["part"] == "frames":
        return None, shard.partition_frames(n, world, case["overlap"])
    r = shard.partition_preloaded(n, world, case["overlap"], case["batch_size"])
    return r, r + [(n, n)] * (world - len(r))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    from svr2_import import load_package
    load_package()
    import torch.distributed as dist
    live = Live()
    eng = stub_engine(live=live)
    shard = mod("shard")
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pipeline = mod("pipeline")
    most = [0]
    run = pipeline.final_slices

    def watched(total, bs, ov, clip_fn, blend_fn, post_fn):      # live kept images at every batch
        def clip(a, b):
            most[0] = max(most[0], live.frames())
            return clip_fn(a, b)
        return run(total, bs, ov, clip, blend_fn, post_fn)

    pipeline.final_slices = watched
    out = []
    for case in grid(world):
        given, _ = ranges_for(case, world)
        reads = []
        v = video(case["total"], 4 if case["kw"]["keep_alpha"] else 3)
        if case["source"] == "open":
            def frames(s, e, v=v):
                reads.append((s, e))
                return odd_chunks(v[s:e], s * 13 + e)
        else:
            frames = v
        most[0] = 0
        got = []
        for first, t in shard.stream_shard(eng, frames, total=case["total"] if case["source"] == "open" else None,
                                           ranges=given, out_dtype=torch.float32 if case["out"] == "f32" else torch.uint8,
                                           batch_size=case["batch_size"], temporal_overlap=case["overlap"],
                                           prepend_frames=case["p"], **case["kw"]):
            got.append((first, t.numpy().copy()))         # by value through the queue
        most[0] = max(most[0], live.frames())
        out.append(dict(got=got, reads=reads, kept=most[0]))
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def contract(eng, case, world):
    """merge_shards of per-rank upscale_video on the video with its mirrored frames in front, the prepend drop, then
    float32 or the CLI's bytes."""
    pipeline, shard = mod("pipeline"), mod("shard")
    from oracle import color_oracle
    v = video(case["total"], 4 if case["kw"]["keep_alpha"] else 3)
    p = case["p"]
    virtual = pipeline.pad_video_temporal(v, count=p, prepend=True) if p else v
    kw = dict(batch_size=case["batch_size"], temporal_overlap=case["overlap"], **case["kw"])
    _, ranges = ranges_for(case, world)
    chunks = [eng.upscale_video(virtual[a:b], prepend_frames=0, **kw) if b > a else None for a, b in ranges]
    like = next(c for c in chunks if c is not None)
    chunks = [like[:0] if c is None else c for c in chunks]
    merged = shard.merge_shards(chunks, case["overlap"],
                                blend=lambda a, b: color_oracle.blend_overlapping_frames(a, b, a.shape[0]))
    if 0 < p < merged.shape[0]:
        merged = merged[p:]
    return merged if case["out"] == "f32" else u8_rule(merged), ranges


def run_world(world, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = dict(q.get(timeout=600) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    return results


@pytest.mark.parametrize("world,port", [(2, 29631), (3, 29632)])
def test_stream_shard_equals_merged_per_rank_upscale(pkg, world, port, monkeypatch):
    results = run_world(world, port)
    eng = stub_engine(monkeypatch.setattr)
    for k, case in enumerate(grid(world)):
        ref, ranges = contract(eng, case, world)
        seen = torch.zeros(ref.shape[0], dtype=torch.int64)
        for rank in range(world):
            res = results[rank][k]
            for first, t in res["got"]:
                t = torch.from_numpy(t)
                assert t.dtype == ref.dtype and torch.equal(t, ref[first:first + t.shape[0]]), (case, rank, first)
                seen[first:first + t.shape[0]] += 1
            a, b = ranges[rank]
            p, total = case["p"], case["total"]
            if case["source"] == "open":                   # reads: the range, plus the mirror's read-ahead
                want = [] if b <= a else [(0, max(b - p, min(p + 1, total)))] if a < p else [(a - p, b - p)]
                assert res["reads"] == want, (case, rank, res["reads"])
            assert res["kept"] <= 2 * case["overlap"], (case, rank, res["kept"])
        assert torch.equal(seen, torch.ones_like(seen)), (case, seen)


def test_merge_plan_matches_merge_shards(pkg):
    """The plan every rank works out from the chunk lengths alone: each output position's value is the frame the plan
    names, or the cross-fade chain it names, exactly as merge_shards computes it."""
    shard = mod("shard")
    for lengths in itertools.product(range(0, 7), repeat=3):
        for ov in range(0, 5):
            chunks = [torch.arange(L, dtype=torch.float32) + 10 * r for r, L in enumerate(lengths)]
            ref = shard.merge_shards([c.view(-1, 1) for c in chunks], ov, blend=lambda a, b: a * 100 + b)
            plan = shard.MergePlan(list(lengths), ov if len(lengths) > 1 else 0)
            assert plan.length == ref.shape[0]
            val = [None] * plan.length
            for r, ps in enumerate(plan.pos):
                for i, j in enumerate(ps):
                    if j is None:
                        continue
                    head = plan.blend[r] is not None and i < ov
                    val[j] = val[j] * 100 + chunks[r][i] if head else chunks[r][i]
            assert torch.equal(torch.stack(val).view(-1, 1) if val else ref, ref), (lengths, ov)
            for r in range(len(lengths)):
                assert len(plan.carry[r]) <= ov


def test_mismatched_ranges_are_refused_before_any_work(pkg, monkeypatch):
    import torch.distributed as dist
    shard = mod("shard")
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    v = video(6)
    read = []
    opener = lambda s, e: read.append((s, e)) or v[s:e]
    for bad in (dict(ranges=[(0, 3), (3, 5)]), dict(ranges=[(0, 3), (4, 6)]), dict(ranges=[(0, 2), (2, 4), (4, 6)]),
                dict(ranges=[(1, 3), (3, 6)]), dict(total=5), dict(out_dtype=torch.bfloat16)):
        with pytest.raises(ValueError):
            shard.stream_shard(object(), v, **bad)
    with pytest.raises(ValueError):
        shard.stream_shard(object(), opener)                     # a reader needs the frame count
    with pytest.raises(ValueError):
        shard.stream_shard(object(), opener, total=6, ranges=[(0, 4), (4, 7)])
    assert read == []
