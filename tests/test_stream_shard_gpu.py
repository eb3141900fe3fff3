"""-m gpu: the rank-seam kernel svr2_blend_overlap_u8 bit for bit against svr2_blend_overlap_f32 and a numpy
restatement of the CLI's bytes, and shard.stream_shard on two ranks (one GPU through gloo; two GPUs through NCCL when
there are two) against the multi-GPU contract, and its per-rank device memory against the video's length."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "comfyui_seedvr2_videoupscaler_b200."


def mod(m):
    return importlib.import_module(NAME + m)


def cli_bytes(v: np.ndarray) -> np.ndarray:
    """The byte of an fp32 value: * 255 in fp32, truncated, saturating, NaN -> 0."""
    with np.errstate(invalid="ignore", over="ignore"):
        b = v.astype(np.float32) * np.float32(255.0)
    return np.where(np.isnan(b), 0, np.clip(b, 0, 255)).astype(np.uint8)


def adversarial_prev(shape, seed):
    """fp32 open-tail values: k / 255 and its neighbours (x 255 lands on or next to an integer), just below and above
    1, above 1, negatives, zeros of both signs, infinities, NaN, and uniform [0, 1) between them."""
    k = np.arange(256, dtype=np.float32) / np.float32(255.0)
    special = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2)),
                              np.array([np.nextafter(np.float32(1), np.float32(0)), 1.0, 1.0000001, 1.5, 255.0, -0.0,
                                        0.0, -1e-8, -0.5, -3.0, np.inf, -np.inf, np.nan], dtype=np.float32)])
    rng = np.random.default_rng(seed)
    v = rng.random(int(np.prod(shape)), dtype=np.float32)
    v[::3] = special[np.arange(v[::3].size) % special.size]
    return torch.from_numpy(v.reshape(shape))


def test_seam_kernel_bitwise(pkg):
    shard = mod("shard")
    all_bf16 = torch.from_numpy(np.arange(65536, dtype=np.uint16).view(np.int16)).view(torch.bfloat16)
    for overlap in range(1, 6):                                    # linear weights below 3, Hann from 3
        for shape in ((1, 65537, 1), (37, 53, 3), (7, 9, 4), (16, 24, 3)):       # odd sizes and a multiple of 4
            n = int(np.prod(shape))
            idx = (torch.arange(overlap * n) * 7919 + 11) % 65536
            cur = all_bf16[idx].view(overlap, *shape).cuda()       # every bf16 value of cur, across the frames
            prev = adversarial_prev((overlap, *shape), overlap * 100 + n).cuda()
            ref = shard.blend_overlap(prev, cur.float())           # svr2_blend_overlap_f32 (padded as it needs)
            f, b = shard.blend_seam(prev, cur, f32=True, u8=True)
            assert torch.equal(f.view(torch.int32), ref.view(torch.int32)), (overlap, shape)
            assert np.array_equal(b.cpu().numpy(), cli_bytes(ref.cpu().numpy())), (overlap, shape)
            f_only, none = shard.blend_seam(prev, cur, f32=True, u8=False)
            none2, b_only = shard.blend_seam(prev, cur, f32=False, u8=True)
            assert none is None and none2 is None
            assert torch.equal(f_only.view(torch.int32), ref.view(torch.int32)) and torch.equal(b_only, b)
            # unaligned buffers: the one-element path
            pb, cb = torch.empty(prev.numel() + 1, device="cuda"), torch.empty(cur.numel() + 1, device="cuda",
                                                                                   dtype=torch.bfloat16)
            pv, cv = pb[1:].view(prev.shape), cb[1:].view(cur.shape)
            pv.copy_(prev)
            cv.copy_(cur)
            f2, b2 = shard.blend_seam(pv, cv, f32=True, u8=True)
            assert torch.equal(f2.view(torch.int32), ref.view(torch.int32)) and torch.equal(b2, b), (overlap, shape)


# ---- two ranks end to end ----------------------------------------------------------------------------------------
def small_engine(pkg, device):
    cfg = mod("dit").dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return mod("pipeline").SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                         pkg.weights.synth_vae_state_dict(seed=2),
                                         torch.randn(58, 64, generator=torch.Generator().manual_seed(3)), device=device)


def contract(eng, video, kw, world, out_dtype):
    """merge_shards of per-rank upscale_video on the video with its mirrored frames in front, the prepend drop, then
    float32 or the CLI's bytes."""
    pipeline, shard = mod("pipeline"), mod("shard")
    p, o = kw.get("prepend_frames", 0), kw["temporal_overlap"]
    virtual = pipeline.pad_video_temporal(video, count=p, prepend=True) if p else video
    opts = {k: v for k, v in kw.items() if k != "prepend_frames"}
    chunks = [eng.upscale_video(virtual[a:b].to(eng.device), **opts)
              for a, b in shard.partition_frames(virtual.shape[0], world, o)]
    merged = shard.merge_shards(chunks, o)
    if 0 < p < merged.shape[0]:
        merged = merged[p:]
    if out_dtype == torch.float32:
        return merged.cpu()
    return torch.nan_to_num(merged * 255.0, nan=0.0).clamp(0, 255).to(torch.uint8).cpu()


CASES = [dict(temporal_overlap=2, color_correction="lab", keep_alpha=True, prepend_frames=2),
         dict(temporal_overlap=3, color_correction="lab", keep_alpha=True, input_noise_scale=0.3)]


def _worker(rank, world, port, backend, job, q):
    sys.path.insert(0, ROOT)
    from svr2_import import load_package
    pkg = load_package()
    import torch.distributed as dist
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group(backend, rank=rank, world_size=world, device_id=dev if backend == "nccl" else None)
    shard = mod("shard")
    out = {}
    try:
        if job == "e2e":
            eng = mod("pipeline").build_synthetic_engine("3b", device=dev)
            g = torch.Generator().manual_seed(7)
            video = torch.rand(17, 36, 52, 4, generator=g)
            for i, case in enumerate(CASES):
                kw = dict(batch_size=5, resolution=72, seed=3, **case)
                for out_dtype in (torch.uint8, torch.float32):
                    src = video if i == 0 else (lambda s, e: iter(video[s:e].split(3)))
                    got = [(first, t) for first, t in shard.stream_shard(eng, src, total=17, out_dtype=out_dtype, **kw)]
                    assert all(t.is_pinned() and t.dtype == out_dtype for _, t in got)
                    ref = contract(eng, video, kw, world, out_dtype)
                    ok = all(torch.equal(t, ref[f:f + t.shape[0]]) for f, t in got)
                    out[(i, str(out_dtype))] = (ok, [(f, t.shape[0]) for f, t in got], ref.shape[0])
        else:
            eng = small_engine(pkg, dev)
            src = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (90, 270, 480, 3), dtype=np.uint8))
            kw = dict(batch_size=5, temporal_overlap=2, resolution=1080, seed=1)

            def peak(n):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                frames = 0
                for _, t in shard.stream_shard(eng, lambda s, e: iter(src[s:e].split(4)), total=n * world, **kw):
                    assert t.shape[1:] == (1080, 1920, 3)
                    frames += t.shape[0]
                torch.cuda.synchronize()
                return torch.cuda.max_memory_allocated() - base, frames

            peak(15)                                                # shapes, tables and the resident workspace
            out["p15"], out["p45"] = peak(15), peak(45)
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_world(world, backend, job, port, timeout=900):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, job, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = dict(q.get(timeout=timeout) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return results


def check_e2e(results, world):
    for key in results[0]:
        total = results[0][key][2]
        seen = np.zeros(total, dtype=np.int64)
        for r in range(world):
            ok, spans, _ = results[r][key]
            assert ok, (key, r)
            for f, n in spans:
                seen[f:f + n] += 1
        assert (seen == 1).all(), (key, seen)


def test_two_ranks_on_one_gpu_through_gloo(pkg):
    check_e2e(run_world(2, "gloo", "e2e", 29641), 2)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_on_two_gpus_through_nccl(pkg):
    check_e2e(run_world(2, "nccl", "e2e", 29642), 2)


def test_per_rank_device_memory_does_not_grow_with_the_video(pkg):
    """1080p output, two ranks on one GPU, batches of 5 with overlap 2: each rank's peak at 45 frames stays within
    32 MiB of its peak at 15 frames."""
    res = run_world(2, "gloo", "memory", 29643)
    for r in range(2):
        (p15, n15), (p45, n45) = res[r]["p15"], res[r]["p45"]
        print(f"rank {r}: peak above the resident state 15 frames/rank {p15 / 2**20:.1f} MiB, "
              f"45 frames/rank {p45 / 2**20:.1f} MiB")
        assert p45 - p15 < 32 * 2 ** 20, (r, p15, p45)
    assert sum(res[r]["p15"][1] for r in range(2)) == 30 and sum(res[r]["p45"][1] for r in range(2)) == 90
