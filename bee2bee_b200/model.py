"""Dense-layer MLP used by the legacy worker tasks (parity:
/root/reference/bee2bee/model.py:7-71 and the manual backprop in node.py:99-182).

Weights are (in_dim, out_dim) like the reference.  ``layer_backward`` returns the same
``dX, gW, gb`` triple the reference's ``layer_backward`` task ships back as JSON.  With a GPU
the forward/backward run on it through ``dense_forward_device`` / ``dense_backward_device``
(bf16 tensor-core GEMM with the bias+activation epilogue for forward when shapes allow)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np

_C = math.sqrt(2.0 / math.pi)


@dataclass
class Layer:
    W: np.ndarray          # (in_dim, out_dim)
    b: np.ndarray          # (out_dim,)
    activation: str        # 'relu' | 'gelu' | 'none'


def act(x: np.ndarray, kind: str) -> np.ndarray:
    if kind == "relu":
        return np.maximum(x, 0)
    if kind == "gelu":
        return 0.5 * x * (1.0 + np.tanh(_C * (x + 0.044715 * x ** 3)))
    return x


def act_derivative(z: np.ndarray, kind: str) -> np.ndarray:
    if kind == "relu":
        return (z > 0).astype(np.float32)
    if kind == "gelu":
        t = np.tanh(_C * (z + 0.044715 * z ** 3))
        return (0.5 * (1.0 + t) + 0.5 * z * (1.0 - t ** 2) * _C * (1.0 + 3 * 0.044715 * z ** 2)).astype(np.float32)
    return np.ones_like(z, dtype=np.float32)


def layer_forward(layer: Layer, x: np.ndarray) -> np.ndarray:
    return act(x @ layer.W + layer.b, layer.activation)


def layer_forward_train(layer: Layer, x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Returns (activation, pre-activation z); the worker caches (x, z) for the backward task."""
    z = x @ layer.W + layer.b
    return act(z, layer.activation), z


def layer_backward(layer: Layer, x: np.ndarray, z: np.ndarray, grad_out: np.ndarray):
    """dX, gW, gb for y = act(xW + b)."""
    gz = grad_out * act_derivative(z, layer.activation)
    return gz @ layer.W.T, x.T @ gz, gz.sum(axis=0)


def random_mlp(input_dim: int, hidden_dim: int, output_dim: int, layers: int, seed: int = 42) -> List[Layer]:
    rng = np.random.default_rng(seed)
    widths = [input_dim] + [hidden_dim] * (layers - 1) + [output_dim]
    out: List[Layer] = []
    for i, (din, dout) in enumerate(zip(widths[:-1], widths[1:])):
        out.append(Layer(W=rng.normal(0.0, 0.02, size=(din, dout)).astype(np.float32),
                         b=np.zeros((dout,), dtype=np.float32),
                         activation="relu" if i < len(widths) - 2 else "none"))
    return out


def serialize_layer(layer: Layer) -> Dict:
    return {"W": layer.W.tolist(), "b": layer.b.tolist(), "activation": layer.activation}


def deserialize_layer(d: Dict) -> Layer:
    return Layer(W=np.asarray(d["W"], dtype=np.float32), b=np.asarray(d["b"], dtype=np.float32),
                 activation=d.get("activation", "none"))


# ------------------------------------------------------------------ device path
def _tc_ok(dev, *dims_128, k: int) -> bool:
    """the wgmma swap-AB GEMM applies: CUDA device, output features multiple of 128, reduction multiple of 64"""
    import torch

    if not str(dev).startswith("cuda") or not torch.cuda.is_available():
        return False
    from . import ops
    return ops.has_native() and all(d % 128 == 0 for d in dims_128) and k % 64 == 0 and k >= 64


def _tc_matmul(a, b_t, bias=None):
    """a [T, K] @ b_t[N, K]^T -> fp32 [T, N] on the wgmma GEMM (bf16 operands, fp32 accumulate, fp32 out)"""
    import torch
    from . import ops

    return ops.gemm(b_t.to(torch.bfloat16).contiguous(), a.to(torch.bfloat16).contiguous(), out_fp32=True,
                    bias=None if bias is None else bias.float().contiguous())


def dense_forward_device(W, b, activation: str, x, device=None):
    """torch tensors in, (y, z) out; runs on ``device`` (GPU when available).  On a H100 with tile-aligned shapes
    the product runs on the wgmma GEMM (bf16 operands, fp32 accumulation, bias fused in the epilogue) -- K12."""
    import torch

    dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
    Wt = torch.as_tensor(W, dtype=torch.float32, device=dev)
    bt = torch.as_tensor(b, dtype=torch.float32, device=dev)
    xt = torch.as_tensor(x, dtype=torch.float32, device=dev)
    if xt.dim() == 2 and _tc_ok(dev, Wt.shape[1], k=Wt.shape[0]):
        z = _tc_matmul(xt, Wt.t(), bt)                      # z[t, out] = sum_in x[t, in] W[in, out] + b[out]
    else:
        z = xt @ Wt + bt
    if activation == "relu":
        y = torch.relu(z)
    elif activation == "gelu":
        y = torch.nn.functional.gelu(z, approximate="tanh")
    else:
        y = z
    return y, z


def dense_backward_device(W, activation: str, x, z, grad_out, device=None):
    import torch

    dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
    Wt = torch.as_tensor(W, dtype=torch.float32, device=dev)
    xt = torch.as_tensor(x, dtype=torch.float32, device=dev)
    zt = torch.as_tensor(z, dtype=torch.float32, device=dev)
    g = torch.as_tensor(grad_out, dtype=torch.float32, device=dev)
    if activation == "relu":
        gz = g * (zt > 0).float()
    elif activation == "gelu":
        t = torch.tanh(_C * (zt + 0.044715 * zt ** 3))
        gz = g * (0.5 * (1 + t) + 0.5 * zt * (1 - t ** 2) * _C * (1 + 3 * 0.044715 * zt ** 2))
    else:
        gz = g
    if xt.dim() == 2 and _tc_ok(dev, Wt.shape[0], Wt.shape[1], k=Wt.shape[1]) and xt.shape[0] % 64 == 0:
        gX = _tc_matmul(gz, Wt)                             # gX[t, in]  = sum_out gz[t, out] W[in, out]
        gW = _tc_matmul(xt.t(), gz.t())                     # gW[in, out] = sum_t x[t, in] gz[t, out]
        return gX, gW, gz.sum(0)
    return gz @ Wt.t(), xt.t() @ gz, gz.sum(0)
