"""Padding-free input bookkeeping (reference: hf_models/utils.py:20-57, model_wrapper/pretraining.py:129-169).

All integer bookkeeping is done on the HOST with numpy (bit-exact with the reference) and shipped with one async
copy, which removes the device->host syncs the reference incurs (`nonzero()`, 0-d CUDA `max_seqlen`;
SURVEY.md section 3.2).
"""

from __future__ import annotations

import math

import numpy as np
import torch


def divide_if_divisible(dividend: int, divisor: int, msg: str) -> int:
    assert dividend % divisor == 0, msg
    return dividend // divisor


def _check_list_type(list_of_list, error_message: str) -> None:
    if list_of_list is None:
        return
    assert isinstance(list_of_list, list), error_message
    assert isinstance(list_of_list[0], list), error_message


def _flatten(x: list[list[int]]) -> np.ndarray:
    y: list[int] = []
    for sequence in x:
        y.extend(sequence)
    return np.asarray(y, dtype=np.int64)


def _to_device(a: np.ndarray, device) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(a))
    if torch.device(device).type == "cuda":
        t = t.pin_memory().to(device, non_blocking=True)
    return t


def convert_padding_free_lists_to_tensors(
    input_ids: list[list[int]] | None = None,
    inputs_embeds: list[list[float]] | None = None,
    position_ids: list[list[int]] | None = None,
    token_type_ids: list[list[int]] | None = None,
    labels: list[list[int]] | None = None,
    device=None,
):
    """Same contract as the reference: returns (input_ids, position_ids, token_type_ids, labels, cu_seqlens,
    max_seqlen); cu_seqlens is int32, everything else int64.  `max_seqlen` is returned as a Python int."""
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    error_message = "{variable} should be of type List[List[{dtype}]]"
    _check_list_type(input_ids, error_message.format(variable="input_ids", dtype="int"))
    _check_list_type(inputs_embeds, error_message.format(variable="inputs_embeds", dtype="float"))
    _check_list_type(position_ids, error_message.format(variable="position_ids", dtype="int"))
    _check_list_type(token_type_ids, error_message.format(variable="token_type_ids", dtype="int"))
    _check_list_type(labels, error_message.format(variable="labels", dtype="int"))
    if inputs_embeds is not None:
        raise NotImplementedError("inputs_embeds is not supported on the B200 padding-free path")
    if token_type_ids is not None:
        raise NotImplementedError("token_type_ids is not supported on the B200 padding-free path")

    seqlens = np.asarray([0] + [len(x) for x in input_ids], dtype=np.int64)
    cu_seqlens = np.cumsum(seqlens).astype(np.int32)
    max_seqlen = int(seqlens.max())
    if position_ids is None:
        position_ids = [list(range(len(x))) for x in input_ids]
    out_pos = _to_device(_flatten(position_ids), device)
    out_ids = _to_device(_flatten(input_ids), device)
    out_labels = _to_device(_flatten(labels), device) if labels is not None else None
    return out_ids, out_pos, None, out_labels, _to_device(cu_seqlens, device), max_seqlen


def prepare_pretraining_inputs_host(
    tokens: np.ndarray, eos_token_id: int | None, reset_attention_mask: bool, reset_position_ids: bool
) -> dict:
    """model_wrapper/pretraining.py:129-169 + :171-194 on the host.  tokens int64 [mbs, seq+1].
    Returns numpy arrays: input_ids [T], labels [T], cu_seqlens int32 [B+1], position_ids, max_seqlen (int)."""
    input_ids = tokens[:, :-1]
    labels = tokens[:, 1:]
    batch_size, sequence_length = input_ids.shape
    flat = np.ascontiguousarray(input_ids).reshape(-1)
    if reset_attention_mask:
        ends = flat == eos_token_id
        ends[sequence_length - 1 :: sequence_length] = True
        cu = np.concatenate([[0], np.nonzero(ends)[0] + 1]).astype(np.int32)
        seqlen = cu[1:] - cu[:-1]
        max_seqlen = int(seqlen.max())
        if reset_position_ids:
            # cat of aranges (reference builds int32 here, pretraining.py:149-152)
            pos = (np.arange(flat.shape[0], dtype=np.int64) - np.repeat(cu[:-1].astype(np.int64), seqlen)).astype(np.int32)
        else:
            pos = np.tile(np.arange(sequence_length, dtype=np.int64), batch_size)
    else:
        cu = np.arange(0, batch_size * sequence_length + 1, sequence_length, dtype=np.int32)
        max_seqlen = sequence_length
        pos = np.tile(np.arange(sequence_length, dtype=np.int64), batch_size)
    return {
        "input_ids": flat,
        "labels": np.ascontiguousarray(labels).reshape(-1),
        "cu_seqlens": cu,
        "position_ids": pos,
        "max_seqlen": max_seqlen,
    }


def resize_vocab_rows(old: torch.Tensor, new_num_tokens: int, lm_head: bool) -> torch.Tensor:
    """One [V, H] matrix of `PreTrainedModel.resize_token_embeddings(new_num_tokens)` (transformers 5.5, mean_resizing=True,
    no pad_to_multiple_of): `old` (fp32, host) -> [new_num_tokens, H].  Rows below min(V, new) are copied; added rows are
    drawn from N(mean, 1e-9 * covariance) of the old rows when that covariance is positive definite, else set to the mean.
    Draws from torch's global CPU generator in transformers' order: the new module's default init first (nn.Embedding:
    normal_; the untied head, an nn.Linear: kaiming_uniform_ = uniform_(-1/sqrt(H), 1/sqrt(H))), then the sample."""
    from torch.distributions import constraints
    from torch.distributions.multivariate_normal import MultivariateNormal

    V, H = old.shape
    if new_num_tokens == V:
        return old
    new = torch.empty(new_num_tokens, H, dtype=old.dtype)
    if lm_head:
        torch.nn.init.kaiming_uniform_(new, a=math.sqrt(5))
    else:
        torch.nn.init.normal_(new)
    if new_num_tokens > V:
        added = new_num_tokens - V
        w = old.to(torch.float32)
        mean = torch.mean(w, axis=0)
        centered = w - mean
        covariance = centered.T @ centered / V
        eps = 1e-9
        if constraints.positive_definite.check(eps * covariance).all():
            new[-added:, :] = MultivariateNormal(mean, covariance_matrix=eps * covariance).sample(
                sample_shape=(added,)).to(old.dtype)
        else:
            new[-added:, :] = mean[None, :].repeat(added, 1).to(old.dtype)
    n = min(V, new_num_tokens)
    new[:n, :] = old[:n, :]
    return new


def resize_vocab_state(sd: dict, new_num_tokens: int) -> dict:
    """`resize_token_embeddings(new_num_tokens)` of a GPTDolomite / MoEDolomite state dict (host fp32 tensors): wte, then
    the untied lm_head (a tied head has no entry of its own); other entries are passed through"""
    out = dict(sd)
    out["transformer.wte.weight"] = resize_vocab_rows(sd["transformer.wte.weight"], new_num_tokens, lm_head=False)
    if "lm_head.weight" in sd:
        out["lm_head.weight"] = resize_vocab_rows(sd["lm_head.weight"], new_num_tokens, lm_head=True)
    return out
