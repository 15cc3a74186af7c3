"""Helpers for the -m gpu tests: raw C-ABI calls on torch-owned device memory."""
import ctypes as C

import torch

from easy_vitpose_b200 import _lib

EPI_BF16, EPI_BF16_GELU, EPI_BF16_RELU_UP, EPI_F32_NCHW, EPI_F32_ADD, EPI_BF16_GELU_ERF = 0, 1, 2, 4, 5, 6
BF16_SENTINEL = 0x7FC1                # a NaN: no GEMM of finite operands stores it
F32_SENTINEL = -0.70710677            # any add of a value of 1e-7 or more changes its bits


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gemm(a, w, bias, out, epi, resid=None, resid_mod=0, aux=(0, 0, 0, 0)):
    m, k = a.shape
    n = w.shape[0]
    _lib.check(_lib.lib().vpb_gemm(ptr(a), ptr(w), ptr(bias), ptr(out), m, n, k, epi, ptr(resid), resid_mod,
                                   aux[0], aux[1], aux[2], aux[3], stream()))
    torch.cuda.synchronize()


def attention(qkv, batch, heads, head_dim=64):
    out = torch.empty((batch * 192, heads * head_dim), dtype=torch.bfloat16, device=qkv.device)
    _lib.check(_lib.lib().vpb_attention(ptr(qkv), batch, heads, head_dim, ptr(out), stream()))
    torch.cuda.synchronize()
    return out


def layernorm(x, g, b, eps=1e-6):
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.check(_lib.lib().vpb_layernorm(ptr(x), ptr(g), ptr(b), ptr(y), x.shape[0], x.shape[1], eps, stream()))
    torch.cuda.synchronize()
    return y


def f32_bits(v):
    return int(torch.tensor([v], dtype=torch.float32).view(torch.int32))


def bits(t):
    """the bit patterns of a bf16 or fp32 tensor"""
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def sentinel_buffer(n, dtype):
    """n elements of bf16 or fp32 holding the sentinel bits, and those bits"""
    b = BF16_SENTINEL if dtype == torch.bfloat16 else f32_bits(F32_SENTINEL)
    return torch.full((n,), b, dtype=torch.int16 if dtype == torch.bfloat16 else torch.int32, device="cuda").view(dtype), b


def untouched(buf, start, stop, sentinel):
    """buf[:start] and buf[stop:] still hold the sentinel bits"""
    v = bits(buf)
    return bool((v[:start] == sentinel).all()) and bool((v[stop:] == sentinel).all())
