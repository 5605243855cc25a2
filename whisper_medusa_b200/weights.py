"""Checkpoint state dict (reference key layout) -> packed engine blob.

The blob layout is owned by the C library (``wm_tensor_info``); this module only knows how each
engine tensor is derived from the HF/reference parameters (SURVEY.md 3.1 step 3):

* q/k/v projections are fused row-wise into one ``[3d, d]`` matrix; the ``head_dim**-0.5`` query
  scaling (HF ``modeling_whisper.py`` ``WhisperAttention.forward``: ``q_proj(x) * scaling``) is NOT
  folded into the weights (that would round fp16-subnormal weights) -- the attention kernels scale
  the scores instead, which is identical because the factor is a power of two;
* ``k_proj`` has no bias (zeros in the fused bias);
* conv weights ``[out, in, kw]`` are re-ordered to ``[out, kw * in]`` for the implicit GEMM over a
  time-major activation (conv1's K = 240 is zero-padded to 256);
* cross-attention k/v projections are fused into ``[2d, d]`` (the encoder-side GEMM writes the
  decode layout ``[pos][k | v]`` directly);
* Medusa head linears are stacked layer-major, ``[L][(K+1) d, d]`` for ``L = medusa_num_layers`` ResBlocks per head
  (reference ``model.py:235-246``); with one layer that is the ``[(K+1) d, d]`` stack of every head.
Matrices stay fp16; vectors (biases, LayerNorm affine) and position tables are stored as fp32.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from . import _lib
from .config import MedusaConfig


def engine_tensors(config: MedusaConfig, sd: Dict[str, torch.Tensor]):
    """Yield ``(engine_name, tensor)`` for every engine tensor."""
    d = config.d_model
    scale = float(config.head_dim) ** -0.5
    if config.head_dim != 64:
        raise NotImplementedError("the CUDA engine supports head_dim 64 only (every Whisper size)")
    if not 1 <= config.medusa_num_layers <= _lib.WM_MAX_HEAD_LAYERS:
        raise NotImplementedError(f"the CUDA engine supports medusa_num_layers 1 .. {_lib.WM_MAX_HEAD_LAYERS}")
    if config.medusa_hidden_size != d:
        raise ValueError("medusa_hidden_size must equal d_model (residual in MedusaResBlock, model.py:210)")

    def f32(k):
        return sd[k].to(torch.float32)

    def f16(k):
        return sd[k].to(torch.float16)

    def fused_qkv(p):
        w = torch.cat([f16(f"{p}.q_proj.weight"), f16(f"{p}.k_proj.weight"), f16(f"{p}.v_proj.weight")], dim=0)
        b = torch.cat([f32(f"{p}.q_proj.bias"), torch.zeros(d), f32(f"{p}.v_proj.bias")])
        return w, b

    enc = "whisper_model.model.encoder"
    c1 = f16(f"{enc}.conv1.weight").permute(0, 2, 1).reshape(d, -1)  # [d, 3*80]
    c1p = torch.zeros(d, 256, dtype=torch.float16)
    c1p[:, : c1.shape[1]] = c1
    yield "enc.conv1_w", c1p
    yield "enc.conv1_b", f32(f"{enc}.conv1.bias")
    yield "enc.conv2_w", f16(f"{enc}.conv2.weight").permute(0, 2, 1).reshape(d, 3 * d).contiguous()
    yield "enc.conv2_b", f32(f"{enc}.conv2.bias")
    yield "enc.pos", f32(f"{enc}.embed_positions.weight")
    for i in range(config.encoder_layers):
        p, e = f"{enc}.layers.{i}", f"enc.{i}."
        yield e + "ln1_g", f32(f"{p}.self_attn_layer_norm.weight")
        yield e + "ln1_b", f32(f"{p}.self_attn_layer_norm.bias")
        w, b = fused_qkv(f"{p}.self_attn")
        yield e + "qkv_w", w
        yield e + "qkv_b", b
        yield e + "o_w", f16(f"{p}.self_attn.out_proj.weight")
        yield e + "o_b", f32(f"{p}.self_attn.out_proj.bias")
        yield e + "ln2_g", f32(f"{p}.final_layer_norm.weight")
        yield e + "ln2_b", f32(f"{p}.final_layer_norm.bias")
        yield e + "fc1_w", f16(f"{p}.fc1.weight")
        yield e + "fc1_b", f32(f"{p}.fc1.bias")
        yield e + "fc2_w", f16(f"{p}.fc2.weight")
        yield e + "fc2_b", f32(f"{p}.fc2.bias")
    yield "enc.lnf_g", f32(f"{enc}.layer_norm.weight")
    yield "enc.lnf_b", f32(f"{enc}.layer_norm.bias")

    dec = "whisper_model.model.decoder"
    yield "dec.embed", f16(f"{dec}.embed_tokens.weight")
    yield "dec.pos", f32(f"{dec}.embed_positions.weight")
    n_dec = config.decoder_layers + (1 if config.is_block else 0)
    for i in range(n_dec):
        p = f"{dec}.layers.{i}" if i < config.decoder_layers else "medusa_block"
        e = f"dec.{i}."
        yield e + "ln1_g", f32(f"{p}.self_attn_layer_norm.weight")
        yield e + "ln1_b", f32(f"{p}.self_attn_layer_norm.bias")
        w, b = fused_qkv(f"{p}.self_attn")
        yield e + "qkv_w", w
        yield e + "qkv_b", b
        yield e + "o_w", f16(f"{p}.self_attn.out_proj.weight")
        yield e + "o_b", f32(f"{p}.self_attn.out_proj.bias")
        yield e + "ln2_g", f32(f"{p}.encoder_attn_layer_norm.weight")
        yield e + "ln2_b", f32(f"{p}.encoder_attn_layer_norm.bias")
        yield e + "cq_w", f16(f"{p}.encoder_attn.q_proj.weight")
        yield e + "cq_b", f32(f"{p}.encoder_attn.q_proj.bias")
        yield e + "ckv_w", torch.cat([f16(f"{p}.encoder_attn.k_proj.weight"), f16(f"{p}.encoder_attn.v_proj.weight")], 0)
        yield e + "ckv_b", torch.cat([torch.zeros(d), f32(f"{p}.encoder_attn.v_proj.bias")])
        yield e + "co_w", f16(f"{p}.encoder_attn.out_proj.weight")
        yield e + "co_b", f32(f"{p}.encoder_attn.out_proj.bias")
        yield e + "ln3_g", f32(f"{p}.final_layer_norm.weight")
        yield e + "ln3_b", f32(f"{p}.final_layer_norm.bias")
        yield e + "fc1_w", f16(f"{p}.fc1.weight")
        yield e + "fc1_b", f32(f"{p}.fc1.bias")
        yield e + "fc2_w", f16(f"{p}.fc2.weight")
        yield e + "fc2_b", f32(f"{p}.fc2.bias")
    yield "dec.lnf_g", f32(f"{dec}.layer_norm.weight")
    yield "dec.lnf_b", f32(f"{dec}.layer_norm.bias")
    nh = config.medusa_num_heads + (0 if config.is_block else 1)
    layers = range(config.medusa_num_layers)
    yield "heads_w", torch.cat([f16(f"medusa_heads.{i}.{l}.linear.weight") for l in layers for i in range(nh)], 0)
    yield "heads_b", torch.cat([f32(f"medusa_heads.{i}.{l}.linear.bias") for l in layers for i in range(nh)], 0)


def pack_blob(handle, config: MedusaConfig, sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Host uint8 tensor of ``wm_weights_nbytes`` bytes laid out as the library dictates."""
    lib = _lib.load()
    nbytes = lib.wm_weights_nbytes(handle)
    blob = torch.zeros(nbytes, dtype=torch.uint8)
    seen = set()
    off, nb, dt = C.c_size_t(), C.c_size_t(), C.c_int32()
    for name, t in engine_tensors(config, sd):
        rc = lib.wm_tensor_info(handle, name.encode(), C.byref(off), C.byref(nb), C.byref(dt))
        if rc != 0:
            raise RuntimeError(f"engine does not know tensor {name}")
        want = torch.float16 if dt.value == 0 else torch.float32
        t = t.to(want).contiguous()
        raw = t.view(torch.uint8).reshape(-1)
        if raw.numel() != nb.value:
            raise ValueError(f"{name}: {raw.numel()} bytes packed, engine expects {nb.value}")
        blob[off.value : off.value + nb.value] = raw
        seen.add(name)
    n = lib.wm_tensor_count(handle)
    names = {lib.wm_tensor_name(handle, i).decode() for i in range(n)}
    if names != seen:
        raise ValueError(f"tensor set mismatch: missing {sorted(names - seen)}, extra {sorted(seen - names)}")
    return blob
