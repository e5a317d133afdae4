"""The serving decode loop of the reference worker on top of the device loop (SURVEY 8 f-1).

``generate_stream`` restates ``ModelWorker.generate_video_stream`` / ``generate_stream`` (valley/serve/model_worker.py:228-297,
:319-426) minus HTTP, logging and file decoding: prompt expansion of ``<video>`` (:338-341), ``max_new_tokens`` cap 1024 (:353),
single-token stop id (:354-360), left truncation to ``context_len - max_new_tokens - 8`` (:367-368), arg-max below temperature
1e-4 else multinomial (:388-395), stop on the stop id or eos (:396-401), and a text update every ``stream_interval`` tokens with
the stop string cut off (:403-412).

What changes is where the loop runs: the reference synchronises device->host on every token (``int(torch.argmax(...))``); here
tokens are produced on the device in chunks of ``stream_interval`` (``vly_generate``: selection, eos/stop-id bookkeeping and early
exit inside the decode step) and the host only looks at the ids when the reference would have emitted text anyway.
The outputs (the sequence of yielded texts) are the same for greedy decoding -- checked in tests against the reference's loop
run token by token through ``forward``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterator, Optional

import torch

from ._lib import VlySampling, check
from .model import (DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_VI_END_TOKEN,
                    DEFAULT_VI_START_TOKEN, DEFAULT_VIDEO_FRAME_TOKEN, sampling_filters)

DEFAULT_VIDEO_TOKEN = "<video>"          # valley/util/config.py


def expand_video_prompt(prompt: str, n_frames: int, use_im_start_end: bool = True) -> str:
    """model_worker.py:338-341: 256 patch tokens, wrapped + T frame tokens when mm_use_im_start_end."""
    replace_token = DEFAULT_IMAGE_PATCH_TOKEN * 256
    if use_im_start_end:
        replace_token = DEFAULT_IM_START_TOKEN + replace_token + DEFAULT_IM_END_TOKEN + DEFAULT_VI_START_TOKEN + \
            DEFAULT_VIDEO_FRAME_TOKEN * n_frames + DEFAULT_VI_END_TOKEN
    return prompt.replace(DEFAULT_VIDEO_TOKEN, replace_token)


def stop_token_index(tokenizer, stop_str: Optional[str]):
    """model_worker.py:354-360: the stop string counts as a stop *id* only if it tokenises to exactly one id."""
    if stop_str is None:
        return None
    ids = tokenizer(stop_str).input_ids
    return ids[0] if len(ids) == 1 else None


def truncate_source(input_ids, context_len: int, max_new_tokens: int):
    """model_worker.py:367-368."""
    max_src_len = context_len - max_new_tokens - 8
    return input_ids[-max_src_len:]


@torch.no_grad()
def generate_stream(model, tokenizer, params: Dict, *, context_len: int = 2048, stream_interval: int = 2) -> Iterator[Dict]:
    """Yields ``{"text": ori_prompt + text_so_far, "error_code": 0}`` exactly when the reference worker does.

    params: "prompt", optional "video" ([T,3,224,224] pixel tensor, already preprocessed -- see valley_b200.video), "temperature"
    (default 1.0), "max_new_tokens" (default 256, capped at 1024), "stop", and "top_k" / "top_p" (HF generate's filters, as
    ``ValleyLlamaForCausalLM.generate`` takes them; absent: no filter)."""
    prompt = params["prompt"]
    ori_prompt = prompt
    video = params.get("video", None)
    images = None
    if video is not None:
        if prompt.count(DEFAULT_VIDEO_TOKEN) != 1:
            raise AssertionError("Number of video does not match number of <video> tokens in prompt")     # :333
        prompt = expand_video_prompt(prompt, video.shape[0], getattr(model.config, "mm_use_im_start_end", False))
        images = video.to(model.device, torch.float16).unsqueeze(0)                                        # :335-336, :345
    temperature = float(params.get("temperature", 1.0))
    top_k, top_p = sampling_filters(params.get("top_k"), params.get("top_p")) if temperature >= 1e-4 else (0, 1.0)
    max_new_tokens = min(int(params.get("max_new_tokens", 256)), 1024)
    stop_str = params.get("stop", None)
    stop_idx = stop_token_index(tokenizer, stop_str)
    input_ids = truncate_source(list(tokenizer(prompt).input_ids), context_len, max_new_tokens)
    eos = getattr(tokenizer, "eos_token_id", None)

    ids = torch.as_tensor([input_ids], dtype=torch.int64, device=model.device)
    S = ids.shape[1]
    if S + max_new_tokens > model.config.max_position_embeddings:
        max_new_tokens = model.config.max_position_embeddings - S
    if max_new_tokens <= 0:
        return
    _, _, _, embeds, _ = model.prepare_inputs_labels_for_multimodal(ids, None, None, None, images)
    cache = model.new_cache(1)
    try:
        logits, _ = model._prefill(cache, embeds, 1)
        sp = VlySampling(temperature if temperature >= 1e-4 else 0.0, int(torch.randint(0, 2 ** 62, (1,)).item()),
                         -1 if eos is None else int(eos), 0, -1 if stop_idx is None else int(stop_idx), top_k, top_p)
        st = torch.cuda.current_stream(model.device).cuda_stream
        tok = torch.empty(1, dtype=torch.int64, device=model.device)
        check(model._lib.vly_sample_logits(model._ctx, cache._h, logits.data_ptr(), C.byref(sp), tok.data_ptr(), st))
        pred_ids = [int(tok.item())]                       # i == 0 is always an emission point (0 % interval == 0)
        chunk = torch.empty(1, max(stream_interval, 1), dtype=torch.int64, device=model.device)
        done = torch.zeros(1, dtype=torch.int32, device=model.device)
        i = 0
        while True:
            token = pred_ids[-1]
            stopped = (stop_idx is not None and token == stop_idx) or (eos is not None and token == eos)
            # i is an emission point: a multiple of the interval, the last token, or a stop (model_worker.py:403)
            cur_out = tokenizer.decode(pred_ids, skip_special_tokens=True)
            if stop_str is not None:
                pos = cur_out.rfind(stop_str)
                if pos != -1:
                    cur_out = cur_out[:pos]
                    stopped = True
            yield {"text": ori_prompt + cur_out, "error_code": 0}
            if stopped or i == max_new_tokens - 1:
                break
            # next emission point: the next multiple of the interval, or the last token
            nxt_i = min((i // stream_interval + 1) * stream_interval, max_new_tokens - 1)
            n = nxt_i - i
            check(model._lib.vly_generate(model._ctx, cache._h, tok.data_ptr(), n, chunk.data_ptr(), C.byref(sp), done.data_ptr(), st))
            k = int(done.item())                            # < n when the stop id / eos ended the row inside the chunk
            got = chunk[0, :k].tolist()
            pred_ids.extend(got)
            i += k
            if k < n:                                       # stopped inside the chunk: emit at the stop, as the reference does
                continue
            tok.copy_(chunk[0, n - 1:n])
    finally:
        cache.release()
