"""Multi-GPU data parallelism for the hot path: one process per GPU, frames sharded over ranks,
ONE all-gather of frame embeddings before pool + projection (BASELINE.json north_star; SURVEY.md 8e).

The reference has no inference-time collective at all (SURVEY.md 2.1); this is new capability.
Every frame's ViT forward is independent (valley_model.py:179-184 loops over batch items), and every
sequence's decode is independent, so the only exchange step is the gather of ``hidden_states[select]``
shards ([F_local,257,1024] bf16) that lets each rank pool/splice the videos it decodes.

``torch.distributed`` (NCCL on GPUs, gloo in the CPU tests) is plumbing.  Two gather paths: ``FusedFrameGather`` (default on
GPUs) -- the last ViT GEMM's epilogue stores every finished tile into every rank's gather buffer over NVLink peer memory, so
compute and collective are one kernel -- and ``encode_frames_sharded`` (local ViT + one ``all_gather_into_tensor``), the plain
baseline the fused path is checked against bit for bit (tests/test_gpu_multi.py, ``bench.py --gpus N``).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced partition of n_items over world ranks: the first (n_items % world) ranks get one extra."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_shard_sizes(n_items: int, world: int) -> List[int]:
    return [shard_bounds(n_items, world, r)[1] - shard_bounds(n_items, world, r)[0] for r in range(world)]


def dealt_frames(n_items: int, world: int, rank: int) -> range:
    """Round-robin ("interleaved") dealing: rank r owns global frames r, r + world, r + 2 world, ...  Every video's frames are
    then spread over all ranks (balanced whatever the per-video frame counts are), so each rank NEEDS remote frames for the
    videos it decodes -- the case the all-gather exists for (BASELINE config 4)."""
    return range(rank, n_items, world)


def dealt_sizes(n_items: int, world: int) -> List[int]:
    return [len(dealt_frames(n_items, world, r)) for r in range(world)]


def gather_frame_features(local_feats: torch.Tensor, n_frames_total: int, group=None, interleaved: bool = False) -> torch.Tensor:
    """All-gather variable-size shards of frame features -> [n_frames_total, tokens, D] on every rank, in global frame order.

    Shards are padded to the largest shard so a single all_gather_into_tensor (one NCCL ncclAllGather)
    moves everything; padding rows are dropped afterwards.  ``interleaved``: shards are ``dealt_frames`` instead of
    contiguous ``shard_bounds`` blocks."""
    world = dist.get_world_size(group)
    if interleaved:
        sizes = dealt_sizes(n_frames_total, world)
        mx = max(sizes)
        assert local_feats.shape[0] == sizes[dist.get_rank(group)], (local_feats.shape, sizes)
        if local_feats.shape[0] < mx:
            pad = torch.zeros(mx - local_feats.shape[0], *local_feats.shape[1:], dtype=local_feats.dtype, device=local_feats.device)
            local_feats = torch.cat([local_feats, pad], 0)
        out = torch.empty(world * mx, *local_feats.shape[1:], dtype=local_feats.dtype, device=local_feats.device)
        dist.all_gather_into_tensor(out, local_feats.contiguous(), group=group)
        # out[r, i] = global frame r + i * world  ->  global order is the (i, r) transpose, minus the padding of the short shards
        return out.view(world, mx, *local_feats.shape[1:]).transpose(0, 1).reshape(world * mx, *local_feats.shape[1:])[:n_frames_total]
    sizes = all_shard_sizes(n_frames_total, world)
    mx = max(sizes)
    assert local_feats.shape[0] == sizes[dist.get_rank(group)], (local_feats.shape, sizes)
    if local_feats.shape[0] < mx:
        pad = torch.zeros(mx - local_feats.shape[0], *local_feats.shape[1:], dtype=local_feats.dtype, device=local_feats.device)
        local_feats = torch.cat([local_feats, pad], 0)
    out = torch.empty(world * mx, *local_feats.shape[1:], dtype=local_feats.dtype, device=local_feats.device)
    dist.all_gather_into_tensor(out, local_feats.contiguous(), group=group)
    if all(s == mx for s in sizes):
        return out
    return torch.cat([out[r * mx: r * mx + sizes[r]] for r in range(world)], 0)


def encode_frames_sharded(encode_fn: Callable[[torch.Tensor], torch.Tensor], local_pixels: torch.Tensor,
                          n_frames_total: int, group=None, interleaved: bool = False) -> torch.Tensor:
    """rank r holds pixels of global frames shard_bounds(n_frames_total, world, r) (or dealt_frames(...) when ``interleaved``);
    returns ALL frame features in global frame order."""
    local = encode_fn(local_pixels) if local_pixels.shape[0] > 0 else \
        torch.zeros(0, 257, 1024, dtype=torch.bfloat16, device=local_pixels.device)
    return gather_frame_features(local, n_frames_total, group, interleaved)


class FusedFrameGather:
    """Fused ViT-encode + all-gather (include/valley_b200.h: vly_gather_* / vly_vit_encode_gather).

    Each rank owns a gather buffer [n_frames_total*257, 1024] bf16 allocated by the library; CUDA IPC handles are
    exchanged once through torch.distributed and mapped by every rank.  ``encode`` then runs the local ViT shard whose
    LAST GEMM epilogue stores each finished tile into every rank's buffer over NVLink (no separate collective kernel),
    followed by a device-side flag exchange.  ``release`` must be enqueued after the consumers of the buffer."""

    def __init__(self, model, n_frames_total: int, group=None):
        import ctypes as C
        from ._lib import check
        self.model, self.group, self.n_frames_total = model, group, n_frames_total
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.tokens = (model.config.vit_image // model.config.vit_patch) ** 2 + 1
        rows = n_frames_total * self.tokens
        buf, handle = C.c_void_p(), C.create_string_buffer(64)
        check(model._lib.vly_gather_create(model._ctx, rows, C.byref(buf), handle))
        handles = [None] * self.world
        dist.all_gather_object(handles, handle.raw, group=group)
        blob = C.create_string_buffer(b"".join(handles), 64 * self.world)
        check(model._lib.vly_gather_open_peers(model._ctx, blob, self.world, self.rank))

        class _Raw:
            __cuda_array_interface__ = {"shape": (rows, model.config.mm_hidden_size), "typestr": "<u2", "data": (buf.value, False), "version": 2}
        self.features = torch.as_tensor(_Raw(), device=model.device).view(torch.bfloat16).view(n_frames_total, self.tokens, model.config.mm_hidden_size)

    def encode(self, local_pixels: torch.Tensor, interleaved: bool = False) -> torch.Tensor:
        """local_pixels: frames shard_bounds(n_frames_total, world, rank) -- or dealt_frames(...) when ``interleaved`` -- ->
        the [n_frames_total,257,1024] buffer (all ranks' features, global frame order)."""
        from ._lib import check
        from .model import _DT
        if interleaved:
            n_local, off, stride = len(dealt_frames(self.n_frames_total, self.world, self.rank)), self.rank, self.world
        else:
            lo, hi = shard_bounds(self.n_frames_total, self.world, self.rank)
            n_local, off, stride = hi - lo, lo, 1
        assert local_pixels.shape[0] == n_local, (local_pixels.shape, n_local)
        px = local_pixels if local_pixels.dtype in _DT else local_pixels.float()
        px = px.to(self.model.device).contiguous()
        check(self.model._lib.vly_vit_encode_gather_strided(
            self.model._ctx, px.data_ptr() if n_local > 0 else None, _DT[px.dtype], n_local, off, stride,
            getattr(self.model.config, "mm_vision_select_layer", -1), torch.cuda.current_stream().cuda_stream))
        return self.features[: self.n_frames_total]      # (the buffer may be larger than this request)

    def release(self):
        from ._lib import check
        check(self.model._lib.vly_gather_release(self.model._ctx, torch.cuda.current_stream().cuda_stream))

    def check(self):
        """Raise if a peer never delivered its rows (the device-side wait timed out): the buffer is stale.  Non-blocking read
        of a pinned flag -- call it after the synchronisation that ends a request."""
        import ctypes as C
        from ._lib import check
        flag = C.c_int(0)
        check(self.model._lib.vly_gather_status(self.model._ctx, C.byref(flag)))


def my_videos(n_videos: int, group=None) -> Tuple[int, int]:
    """Videos whose sequences this rank decodes (LLM replicated per GPU, batch sharded; no further collective)."""
    return shard_bounds(n_videos, dist.get_world_size(group), dist.get_rank(group))


def generate_sharded(model, input_ids: torch.Tensor, local_pixels: torch.Tensor, n_videos: int, n_frames: int,
                     max_new_tokens: int, group=None, fused: "FusedFrameGather | None" = None, interleaved: bool = False) -> torch.Tensor:
    """Config-4 style request: ``n_videos`` videos x ``n_frames`` frames, frames sharded over ranks for the ViT
    (contiguous blocks, or dealt round-robin when ``interleaved``), one all-gather, then every rank pools/projects/splices and
    greedy-decodes its own videos.  ``input_ids`` [n_videos_local, S] are this rank's prompts; returns this rank's generated ids."""
    if fused is not None:
        feats = fused.encode(local_pixels, interleaved)       # ViT + gather in one pass over NVLink
    else:
        feats = encode_frames_sharded(model.encode_frames, local_pixels, n_videos * n_frames, group, interleaved)   # plain NCCL all-gather
    lo, hi = my_videos(n_videos, group)
    mine = feats.view(n_videos, n_frames, *feats.shape[1:])[lo:hi].reshape((hi - lo) * n_frames, *feats.shape[1:]).contiguous()
    B = hi - lo
    _, _, _, embeds, _ = model.prepare_inputs_labels_for_multimodal(input_ids, None, None, None, None,
                                                                    frame_features=mine, n_frames=n_frames)
    if fused is not None:
        fused.release()                                       # the gather buffer has been consumed (stream order)
    cache = model.new_cache(B)
    try:
        S = input_ids.shape[1]
        out = model._generate_with_cache(cache, input_ids, embeds, max_new_tokens, False, 1.0, None, None)[:, S:]
    finally:
        cache.release()
    if fused is not None:
        fused.check()          # a timed-out gather of an EARLIER request is reported here at the latest (pinned flag, no sync)
    return out
