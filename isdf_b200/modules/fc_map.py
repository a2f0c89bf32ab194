"""SDF MLP -- host-side mirror of reference isdf/modules/fc_map.py.

`SDFMap` keeps the reference's module tree (so `state_dict()` names/shapes and the random
initialisation under a given torch seed are identical: in_layer.0, mid1.i.0, cat_layer.0, mid2.i.0,
out_alpha) but its parameters are views into ONE flat fp32 buffer, which is what the CUDA kernels
(re-pack, fused forward/backward, AdamW) consume.  forward() runs the fused PE+MLP kernel (K2); when
the input requires grad it runs K3 and also yields d sdf / d x, which `gradient()` hands back --
the reference obtains the same tensor with autograd (fc_map.py:12-22).
"""
import os

import numpy as np
import torch
import torch.nn as nn

import warnings

from .. import DEFAULT_PRECISION, _lib
from ..engine import Engine


def gradient(inputs, outputs):
    """d outputs / d inputs for outputs produced by SDFMap.forward(inputs) (fc_map.py:12-22)."""
    g = getattr(outputs, "_isdf_input_grad", None)
    if g is not None and getattr(outputs, "_isdf_input", None) is inputs:
        return g
    ones = torch.ones_like(outputs, requires_grad=False)
    return torch.autograd.grad(outputs, inputs, grad_outputs=ones, create_graph=True, retain_graph=True,
                               only_inputs=True)[0]


def chunks(pc, chunk_size, fc_sdf_map, to_cpu=False):
    """Evaluate fc_sdf_map over pc [N,3] in slices of chunk_size (fc_map.py:25-48)."""
    outs = []
    for start in range(0, pc.shape[0], chunk_size):
        a = fc_sdf_map(pc[start:start + chunk_size, :]).squeeze(dim=-1)
        outs.append(a.cpu() if to_cpu else a)
    return torch.cat(outs, dim=-1)


def fc_block(in_f, out_f):
    return nn.Sequential(nn.Linear(in_f, out_f), nn.Softplus(beta=100))


def init_weights(m, init_fn=nn.init.xavier_normal_):
    if isinstance(m, nn.Linear):
        init_fn(m.weight)


class _SdfWithGrad(torch.autograd.Function):
    """sdf = f(x); backward gives d/dx only (= g * grad_out).  Parameter gradients of the training
    loss come from the fused kernel (Trainer.sdf_eval_and_loss), not from autograd."""

    @staticmethod
    def forward(ctx, x, sdf, g):
        ctx.save_for_backward(g)
        return sdf.clone()

    @staticmethod
    def backward(ctx, grad_out):
        (g,) = ctx.saved_tensors
        return g * grad_out[..., None], None, None


class SDFMap(nn.Module):
    def __init__(self, positional_encoding, hidden_size=256, hidden_layers_block=1, scale_output=1.):
        super().__init__()
        self.scale_output = scale_output
        self.positional_encoding = positional_encoding
        e = positional_encoding.embedding_size
        self.hidden_size, self.hidden_layers_block = hidden_size, hidden_layers_block
        self.in_layer = fc_block(e, hidden_size)
        self.mid1 = nn.Sequential(*[fc_block(hidden_size, hidden_size) for _ in range(hidden_layers_block)])
        self.cat_layer = fc_block(hidden_size + e, hidden_size)
        self.mid2 = nn.Sequential(*[fc_block(hidden_size, hidden_size) for _ in range(hidden_layers_block)])
        self.out_alpha = nn.Linear(hidden_size, 1)
        self.apply(init_weights)
        self.precision = os.environ.get("ISDFB_PRECISION", DEFAULT_PRECISION)
        self.max_points = int(os.environ.get("ISDFB_MAX_POINTS", 32768))
        self._engine = None
        self._engine_precision = self._engine_tr_key = None
        self._flat = None
        self._packed_sig = None

    # ---- flat parameter storage ------------------------------------------------------
    def flat_parameters(self):
        """The single contiguous fp32 buffer all parameters are views of (re-built if views broke)."""
        ps = list(self.parameters())
        ok = self._flat is not None and self._flat.device == ps[0].device
        if ok:
            off = 0
            base = self._flat.data_ptr()
            for p in ps:
                if p.data_ptr() != base + 4 * off or not p.is_contiguous():
                    ok = False
                    break
                off += p.numel()
        if not ok:
            flat = torch.cat([p.detach().reshape(-1).float() for p in ps]).contiguous()
            off = 0
            for p in ps:
                p.data = flat[off:off + p.numel()].view_as(p)
                off += p.numel()
            self._flat = flat
            self._packed_sig = None
        return self._flat

    def engine(self):
        flat = self.flat_parameters()
        dev = flat.device
        pe = self.positional_encoding
        tr_key = pe.transform          # identity, not value: this runs on every call and must not touch the device
        if (self._engine is None or self._engine.device != dev or self._engine_precision != self.precision
                or self._engine_tr_key is not tr_key):
            try:
                self._engine = Engine(dev, pe.n_freqs, self.hidden_size, self.hidden_layers_block, pe.scale,
                                      self.scale_output, transform=pe.transform, precision=self.precision,
                                      max_points=self.max_points)
            except _lib.IsdfbError as e:
                if self.precision == "fp32" or "tensor-core path supports" not in str(e):
                    raise
                # shapes the tensor-core (wgmma) kernels do not take run on the CUDA-core fp32 kernels of the same library
                warnings.warn("isdf_b200: %s -- using precision 'fp32' (CUDA-core kernels) for this model" % e)
                self._engine = Engine(dev, pe.n_freqs, self.hidden_size, self.hidden_layers_block, pe.scale,
                                      self.scale_output, transform=pe.transform, precision="fp32",
                                      max_points=self.max_points)
            self._engine_precision, self._engine_tr_key = self.precision, tr_key
            self._packed_sig = None
        sig = (flat.data_ptr(), tuple(p._version for p in self.parameters()))
        if sig != self._packed_sig:
            self._engine.pack_weights(flat)
            self._packed_sig = sig
        return self._engine

    def mark_packed(self):
        """Called by the fused optimiser after it updated the flat buffer AND re-packed in-kernel."""
        self._packed_sig = (self._flat.data_ptr(), tuple(p._version for p in self.parameters()))

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in ("_engine", "_flat", "_packed_sig", "_engine_precision", "_engine_tr_key"):
                new.__dict__[k] = None
            else:
                new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    # ---- forward -----------------------------------------------------------------------
    def forward(self, x, noise_std=None, pe_mask=None, sdf1=None):
        if pe_mask is not None:
            raise NotImplementedError("pe_mask is not supported by the fused kernels (unused by every shipped "
                                      "reference config)")
        eng = self.engine()
        xd = x.detach()
        noise = None
        if noise_std is not None:
            noise = torch.randn(x.shape[:-1], device=x.device)       # same draw as fc_map.py:106-108
        want = x.requires_grad and torch.is_grad_enabled()
        if not want:
            return eng.forward(xd, noise=noise, noise_std=noise_std or 0.0)
        sdf, g = eng.forward(xd, noise=noise, noise_std=noise_std or 0.0, want_grad=True)
        out = _SdfWithGrad.apply(x, sdf, g)
        out._isdf_input_grad = g
        out._isdf_input = x
        return out
