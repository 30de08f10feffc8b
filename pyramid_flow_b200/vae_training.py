"""Trainable causal 3-D convolution, and its drop-in for the reference's causal video VAE training step.

`causal_conv3d(x, weight, bias, stride)` has the semantics of the reference's CausalConv3d.forward with temporal_chunk=False
(video_vae/modeling_causal_conv.py:116-126): 2 zero frames in front, 1 zero pixel on each side of H and W (kernels 3x3x3;
1x1x1 convs pad nothing), then nn.Conv3d(padding=0) with stride 1, (1,2,2) or (2,1,1).  It is an autograd function on the
library's kernels (include/pf_b200.h):
  forward : pf_conv3d_pack (x -> channels-last bf16 with the causal frames, kept for the backward), pf_causal_conv3d;
            the output is an NCDHW view of the channels-last result (memory format channels_last_3d, no copy);
  backward: pf_conv3d_pack of dy (dilated along strided axes, the bias gradient from the same pass), then
            dx = pf_causal_conv3d on the packed dy with the flipped, transposed filter (only if x needs a gradient) and
            dW = pf_conv3d_wgrad (only if the weight needs one).
Operands are rounded to bf16 (as under autocast) and accumulated in fp32; dW and db are computed in fp32, dx has x's dtype,
the output is bf16 under bf16 autocast and x's dtype otherwise.  Every reduction has a fixed order, so the bits do not
change between runs or under torch.utils.checkpoint recompute.  The packed input is saved with save_for_backward, so
saved-tensor hooks (non-reentrant checkpointing, save_on_cpu) manage it; the backward frees nothing, so it can run more
than once on one graph (LPIPSWithDiscriminator's adaptive weight takes torch.autograd.grad of the last layer's weight with
retain_graph=True before the real backward, video_vae/modeling_loss.py:89-96).

`install_training_convs(vae)` patches the `forward` of every CausalConv3d of a reference CausalVideoVAE (or of the `.vae`
of a CausalVideoVAELossWrapper) in place; everything else of the training step -- GroupNorm, SiLU, the mid-block attention,
the up-samplers' rearranges, LPIPS and the discriminator -- stays torch.  `uninstall_training_convs` restores the instances.

`causal_group_norm(x, weight, bias, num_groups, eps, silu)` is CausalGroupNorm.forward (video_vae/modeling_causal_conv.py:36-43:
GroupNorm of every (batch, frame)), optionally followed by a SiLU, as an autograd function on pf_groupnorm_train_fwd / _bwd.
x (bf16 or fp32) is read in place when it is channels_last_3d (what causal_conv3d returns) or has contiguous (h, w) planes
(NCDHW, the up-samplers' rearranged copies); any other layout is copied to channels_last_3d first (counted in
`layout_copies`).  The output has x's form; its dtype is fp32 under autocast (torch's group_norm autocasts to fp32) and x's
dtype otherwise, or `out_dtype`.  Saved are x itself and the fp32 per-frame (mean, rstd); the backward recomputes the
normalised value, and its partial sums are added in a fixed order (the bits repeat, also under checkpoint recompute).  If a
saved-tensor hook returns x in other strides (save_on_cpu does), the backward copies it back into the forward's form.  Where
x has planes and the gradient arrives channels-last (the sites after the up-samplers), the backward repacks a bf16 x
channels-last with pf_conv3d_pack and runs the channel-form kernels.
`install_training_norms(vae)` runs every CausalGroupNorm with its following SiLU fused (the SiLU module is replaced by
nn.Identity on the instance) and, under bf16 autocast, a bf16 output: every such output feeds a conv that rounds its input
to bf16 anyway.  `uninstall_training_norms` restores the module tree.  The two installs compose in either order.
"""
from __future__ import annotations

import types
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib, ops

STRIDES = ((1, 1, 1), (1, 2, 2), (2, 1, 1))
KERNELS = ((1, 1, 1), (3, 3, 3))
_MARK = "_pf_training_conv"


def _pad64(c: int) -> int:
    return (c + 63) // 64 * 64


def forward_filter(weight: torch.Tensor, cout_p: int, cin_p: int) -> torch.Tensor:
    """[Cout, Cin, kt, kh, kw] -> bf16 [cout_p, taps*cin_p], K index tap*cin_p + ci (pf_causal_conv3d's layout)."""
    cout, cin = weight.shape[:2]
    wf = torch.zeros(cout_p, *weight.shape[2:], cin_p, device=weight.device, dtype=torch.bfloat16)
    wf[:cout, ..., :cin] = weight.detach().permute(0, 2, 3, 4, 1)
    return wf.reshape(cout_p, -1)


def dgrad_filter(weight: torch.Tensor, cout_p: int, cin_p: int) -> torch.Tensor:
    """The data gradient's filter: flipped on all three axes, Cin and Cout swapped: bf16 [cin_p, taps*cout_p]."""
    cout, cin = weight.shape[:2]
    wb = torch.zeros(cin_p, *weight.shape[2:], cout_p, device=weight.device, dtype=torch.bfloat16)
    wb[:cin, ..., :cout] = weight.detach().flip(2, 3, 4).permute(1, 2, 3, 4, 0)
    return wb.reshape(cin_p, -1)


def _out_dims(x_shape, stride) -> Tuple[int, int, int]:
    _, _, t, h, w = x_shape
    st, sh, sw = stride
    return (t - 1) // st + 1, h // sh, w // sw


class _CausalConv3d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride, out_dtype):
        cout, cin, kt, kh, kw = weight.shape
        b, _, t, h, w = x.shape
        to, ho, wo = _out_dims(x.shape, stride)
        cin_p, cout_p = _pad64(cin), _pad64(cout)
        # the packed input holds exactly the frames the conv reads: (to-1)*st + kt (a stride-2 conv over an even number of
        # frames never reads the last one)
        t_in = (to - 1) * stride[0] + kt
        xp = torch.empty(b, t_in, h, w, cin_p, device=x.device, dtype=torch.bfloat16)
        ops.conv3d_pack(x[:, :, :t_in - (kt - 1)], xp, t_offset=kt - 1)
        bias_p = None
        if bias is not None:
            bias_p = torch.zeros(cout_p, device=x.device, dtype=torch.float32)
            bias_p[:cout] = bias.detach()
        y = torch.empty(b, to, ho, wo, cout, device=x.device, dtype=out_dtype)
        ops.causal_conv3d(xp, forward_filter(weight, cout_p, cin_p), bias_p, y, kernel=(kt, kh, kw), stride=stride)
        # through save_for_backward, so that saved-tensor hooks see the packed input: non-reentrant checkpointing (the
        # reference encoder's, video_vae/modeling_enc_dec.py:170-178) drops it after the forward, save_on_cpu moves it
        ctx.save_for_backward(weight, xp)
        ctx.stride, ctx.x_shape, ctx.x_dtype, ctx.has_bias = stride, tuple(x.shape), x.dtype, bias is not None
        return y.permute(0, 4, 1, 2, 3)

    @staticmethod
    def backward(ctx, dy):
        weight, xp = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        cout, cin, kt, kh, kw = weight.shape
        b, _, t, h, w = ctx.x_shape
        stride = ctx.stride
        cin_p, cout_p = _pad64(cin), _pad64(cout)
        # dy with zeros inserted along the strided axes and kt-1 zero frames at the end: the data gradient's input, and
        # what the weight gradient reads (every stride-th element)
        dyp = torch.empty(b, t + kt - 1, h, w, cout_p, device=dy.device, dtype=torch.bfloat16)
        db = torch.empty(cout, device=dy.device, dtype=torch.float32) if (need_b and ctx.has_bias) else None
        ops.conv3d_pack(dy, dyp, t_offset=0, dil=stride, bias_grad=db)
        dx = dw = None
        if need_x:
            dxc = torch.empty(b, t, h, w, cin, device=dy.device, dtype=ctx.x_dtype)
            ops.causal_conv3d(dyp, dgrad_filter(weight, cout_p, cin_p), None, dxc, kernel=(kt, kh, kw))
            dx = dxc.permute(0, 4, 1, 2, 3)
        if need_w:
            dw = torch.empty(weight.shape, device=dy.device, dtype=torch.float32)
            ops.conv3d_wgrad(xp, dyp, dw, out_shape=_out_dims(ctx.x_shape, stride), stride=stride)
            dw = dw.to(weight.dtype)
        if db is not None:
            db = db.to(weight.dtype)
        return dx, dw, db, None, None


def _check_geometry(x: torch.Tensor, weight: torch.Tensor, stride) -> None:
    if x.dim() != 5 or weight.dim() != 5 or x.shape[1] != weight.shape[1]:
        raise ValueError(f"causal_conv3d: x {tuple(x.shape)} and weight {tuple(weight.shape)} are not [B, Cin, T, H, W] / "
                         "[Cout, Cin, kt, kh, kw]")
    if tuple(weight.shape[2:]) not in KERNELS:
        raise ValueError(f"causal_conv3d: kernel {tuple(weight.shape[2:])} is not 1x1x1 or 3x3x3")
    if stride not in STRIDES or (stride != (1, 1, 1) and tuple(weight.shape[2:]) != (3, 3, 3)):
        raise ValueError(f"causal_conv3d: stride {stride} is not one of {STRIDES} (strided convs are 3x3x3)")
    if x.dtype not in (torch.bfloat16, torch.float32):
        raise TypeError(f"causal_conv3d: x must be bf16 or fp32, got {x.dtype}")
    if stride[1] == 2 and (x.shape[3] % 2 or x.shape[4] % 2):
        raise ValueError(f"causal_conv3d: a spatial stride-2 conv needs even H and W, got {tuple(x.shape[3:])}")
    if not (x.is_cuda and weight.is_cuda):
        raise RuntimeError("causal_conv3d runs on the library's CUDA kernels: x and weight must be CUDA tensors "
                           "(there is no CPU path)")


def causal_conv3d(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, stride=(1, 1, 1)) -> torch.Tensor:
    """CausalConv3d.forward (temporal_chunk=False) of x [B, Cin, T, H, W] with an nn.Conv3d's weight / bias / stride."""
    stride = (stride,) * 3 if isinstance(stride, int) else tuple(int(s) for s in stride)
    _check_geometry(x, weight, stride)
    _lib.require_device()
    bf16_autocast = torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16
    out_dtype = torch.bfloat16 if bf16_autocast else x.dtype
    return _CausalConv3d.apply(x, weight, bias, stride, out_dtype)


# ---------------------------------------------------------------------------------------------------------------- drop-in
def _target(vae) -> nn.Module:
    inner = getattr(vae, "vae", None)         # CausalVideoVAELossWrapper.vae (video_vae/causal_video_vae_wrapper.py:42)
    return inner if isinstance(inner, nn.Module) else vae


def causal_convs(vae) -> List[Tuple[str, nn.Module]]:
    """(name, module) of every reference CausalConv3d under a CausalVideoVAE or a CausalVideoVAELossWrapper's `.vae`."""
    return [(n, m) for n, m in _target(vae).named_modules()
            if type(m).__name__ == "CausalConv3d" and isinstance(getattr(m, "conv", None), nn.Conv3d)]


def _patched_forward(self, x, is_init_image=True, temporal_chunk=False):
    if temporal_chunk:
        raise ValueError("the training convolutions do not run the temporal-chunk feature cache (the reference asserts it "
                         "is inference only); use B200CausalVAE for chunked encode / decode")
    return causal_conv3d(x, self.conv.weight, self.conv.bias, self.conv.stride)


def _refusal(name: str, m: nn.Module) -> Optional[str]:
    c = m.conv
    if tuple(c.kernel_size) not in KERNELS:
        return f"{name}: kernel {tuple(c.kernel_size)} is not 1x1x1 or 3x3x3"
    if tuple(c.stride) not in STRIDES or (tuple(c.stride) != (1, 1, 1) and tuple(c.kernel_size) != (3, 3, 3)):
        return f"{name}: stride {tuple(c.stride)} is not one of {STRIDES}"
    if tuple(c.dilation) != (1, 1, 1):
        return f"{name}: dilation {tuple(c.dilation)} is not 1"
    if c.groups != 1 or tuple(c.padding) != (0, 0, 0) or c.padding_mode != "zeros":
        return f"{name}: grouped or self-padding Conv3d"
    if getattr(m, "pad_mode", "constant") != "constant":
        return f"{name}: pad_mode {m.pad_mode!r} is not 'constant'"
    return None


def install_training_convs(vae) -> None:
    """Run every CausalConv3d of a reference CausalVideoVAE (or CausalVideoVAELossWrapper) on `causal_conv3d`."""
    convs = causal_convs(vae)
    if not convs:
        raise ValueError("no CausalConv3d found: pass a reference CausalVideoVAE or CausalVideoVAELossWrapper")
    cp_initialized = type(convs[0][1]).forward.__globals__.get("is_context_parallel_initialized")
    if cp_initialized is not None and cp_initialized():
        raise ValueError("a context-parallel group is initialised: CausalConv3d.context_parallel_forward (the stage-2 "
                         "recipe) is not replaced by the training convolutions")
    for name, m in convs:
        why = _refusal(name, m)
        if why is not None:
            raise ValueError(f"install_training_convs: {why}")
    for _, m in convs:
        m.forward = types.MethodType(_patched_forward, m)
        setattr(m, _MARK, True)


def uninstall_training_convs(vae) -> None:
    for _, m in causal_convs(vae):
        if m.__dict__.pop(_MARK, False):
            del m.forward


# ------------------------------------------------------------------------------------------------------------- GroupNorm
layout_copies = 0     # inputs / gradients causal_group_norm had to copy into a layout the kernels read
_checked_devices = set()


def _require_device_once() -> None:
    """_lib.require_device() (a cudaGetDeviceProperties, about 3 ms) once per device: the op runs at every norm site."""
    dev = torch.cuda.current_device()
    if dev not in _checked_devices:
        _lib.require_device()
        _checked_devices.add(dev)


def _bf16_autocast() -> bool:
    return torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16


def _in_form(t: torch.Tensor, form: Optional[str]) -> torch.Tensor:
    """t in the layout form `form` (or channels_last_3d if form is None / t is in neither form)."""
    global layout_copies
    have = ops.groupnorm_form(t)
    if have is not None and (form is None or have == form):
        return t
    layout_copies += 1
    if form == "plane":
        return t.contiguous()
    return t.contiguous(memory_format=torch.channels_last_3d)


def _channels_last_for(x: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    """x in channel form when x has planes and dy arrives channels-last (the next conv's data gradient does, at the sites
    after the up-samplers): a bf16 x with channels a multiple of 64 is repacked by pf_conv3d_pack (an exact, vectorised
    transposing copy), which is far cheaper than torch's permuting copy of dy into planes."""
    global layout_copies
    if not (ops.groupnorm_form(x) == "plane" and ops.groupnorm_form(dy) == "channel" and x.dtype == torch.bfloat16
            and x.shape[1] % 64 == 0):
        return x
    layout_copies += 1
    b, c, t, h, w = x.shape
    xc = torch.empty(b, t, h, w, c, device=x.device, dtype=torch.bfloat16)
    ops.conv3d_pack(x, xc, t_offset=0)
    return xc.permute(0, 4, 1, 2, 3)


def _empty_in_form(like: torch.Tensor, form: str, dtype: torch.dtype) -> torch.Tensor:
    if form == "channel":
        b, c, t, h, w = like.shape
        return torch.empty(b, t, h, w, c, device=like.device, dtype=dtype).permute(0, 4, 1, 2, 3)
    return torch.empty(like.shape, device=like.device, dtype=dtype)


class _CausalGroupNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, groups, eps, silu, out_dtype):
        x = _in_form(x, None)
        form = ops.groupnorm_form(x)
        b, c, t = x.shape[:3]
        gamma, beta = weight.detach().float().contiguous(), bias.detach().float().contiguous()
        stats = torch.empty(b * t, groups, 2, device=x.device, dtype=torch.float32)
        y = _empty_in_form(x, form, out_dtype)
        ops.groupnorm_train_fwd(x, gamma, beta, stats, y, groups=groups, eps=eps, silu=silu)
        # through save_for_backward, so that saved-tensor hooks (non-reentrant checkpointing, save_on_cpu) see x and the
        # statistics; nothing activation-sized besides x is kept
        ctx.save_for_backward(x, weight, bias, stats)
        ctx.groups, ctx.silu, ctx.form = groups, silu, form
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, stats = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        # a saved-tensor hook may hand x back with other strides than it had in the forward (save_on_cpu unpacks into a
        # contiguous NCDHW tensor): it is brought back to the forward's form, so the backward runs the same kernels, in the
        # same summation order, as without the hook
        x = _in_form(x, ctx.form)
        x = _channels_last_for(x, dy)
        form = ops.groupnorm_form(x)
        dy = _in_form(dy, form)
        gamma, beta = weight.detach().float().contiguous(), bias.detach().float().contiguous()
        dx = _empty_in_form(x, form, x.dtype) if need_x else None
        c = x.shape[1]
        dgamma = torch.empty(c, device=x.device, dtype=torch.float32) if need_w else None
        dbeta = torch.empty(c, device=x.device, dtype=torch.float32) if need_b else None
        ops.groupnorm_train_bwd(x, dy, gamma, beta, stats, dx, dgamma, dbeta, groups=ctx.groups, silu=ctx.silu)
        if dgamma is not None:
            dgamma = dgamma.to(weight.dtype)
        if dbeta is not None:
            dbeta = dbeta.to(bias.dtype)
        return dx, dgamma, dbeta, None, None, None, None


def causal_group_norm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, num_groups: int, eps: float,
                      silu: bool = False, out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """CausalGroupNorm.forward of x [B, C, T, H, W] (then SiLU if `silu`) with an affine GroupNorm's weight / bias.
    out_dtype None: fp32 under autocast (as torch's group_norm), x's dtype otherwise."""
    if x.dim() != 5 or weight is None or bias is None or weight.shape != (x.shape[1],) or bias.shape != (x.shape[1],):
        raise ValueError(f"causal_group_norm: x {tuple(x.shape)} is not [B, C, T, H, W] with an affine weight / bias of C")
    if x.dtype not in (torch.bfloat16, torch.float32):
        raise TypeError(f"causal_group_norm: x must be bf16 or fp32, got {x.dtype}")
    c = x.shape[1]
    if c % 8 or c % num_groups:
        raise ValueError(f"causal_group_norm: {c} channels must be a multiple of 8 and of num_groups={num_groups}")
    if not (x.is_cuda and weight.is_cuda and bias.is_cuda):
        raise RuntimeError("causal_group_norm runs on the library's CUDA kernels: x, weight and bias must be CUDA tensors "
                           "(there is no CPU path)")
    if out_dtype is None:
        out_dtype = torch.float32 if torch.is_autocast_enabled("cuda") else x.dtype
    if out_dtype not in (torch.bfloat16, torch.float32):
        raise TypeError(f"causal_group_norm: out_dtype must be bf16 or fp32, got {out_dtype}")
    _require_device_once()
    return _CausalGroupNorm.apply(x, weight, bias, int(num_groups), float(eps), bool(silu), out_dtype)


# ---------------------------------------------------------------------------------------------------------------- drop-in
_NORM_MARK = "_pf_training_norm"
_SAVED_ACT = "_pf_saved_activation"


def causal_group_norms(vae) -> List[Tuple[str, nn.Module]]:
    """(name, module) of every reference CausalGroupNorm under a CausalVideoVAE or a CausalVideoVAELossWrapper's `.vae`."""
    return [(n, m) for n, m in _target(vae).named_modules()
            if type(m).__name__ == "CausalGroupNorm" and isinstance(m, nn.GroupNorm)]


def _norm_sites(vae):
    """(owner, activation attribute, [its CausalGroupNorms]) for every norm -> SiLU pair the install fuses:
    CausalResnetBlock3D norm1 / norm2 -> nonlinearity, and the encoder's / decoder's conv_norm_out -> conv_act."""
    sites = []
    for name, m in _target(vae).named_modules():
        if type(m).__name__ == "CausalResnetBlock3D":
            sites.append((name, m, "nonlinearity", [getattr(m, "norm1", None), getattr(m, "norm2", None)]))
        elif type(getattr(m, "conv_norm_out", None)).__name__ == "CausalGroupNorm" and hasattr(m, "conv_act"):
            sites.append((name, m, "conv_act", [m.conv_norm_out]))
    return sites


def _norm_refusal(name: str, owner: nn.Module, act_attr: str, norms) -> Optional[str]:
    act = owner.__dict__.get(_SAVED_ACT, getattr(owner, act_attr))
    if type(act) is not nn.SiLU:
        return f"{name}.{act_attr} is {type(act).__name__}, not nn.SiLU"
    if act_attr == "nonlinearity":
        if getattr(owner, "time_embedding_norm", "default") != "default":
            return f"{name}: time_embedding_norm {owner.time_embedding_norm!r} is not 'default'"
        drop = getattr(owner, "dropout", None)
        if drop is not None and getattr(drop, "p", 0.0) > 0:
            return f"{name}: dropout p={drop.p} sits between the norm's bf16 output and conv2"
    for n in norms:
        if type(n).__name__ != "CausalGroupNorm":
            return f"{name}: {type(n).__name__} before the {act_attr} is not a CausalGroupNorm"
        if not n.affine:
            return f"{name}: a CausalGroupNorm without affine parameters"
        if n.num_channels % 8:
            return f"{name}: {n.num_channels} channels are not a multiple of 8"
    return None


def _patched_norm_forward(self, x):
    return causal_group_norm(x, self.weight, self.bias, self.num_groups, self.eps, silu=True,
                             out_dtype=torch.bfloat16 if _bf16_autocast() else None)


def install_training_norms(vae) -> None:
    """Run every CausalGroupNorm of a reference CausalVideoVAE (or CausalVideoVAELossWrapper) on `causal_group_norm` with
    the SiLU after it fused; the SiLU module becomes nn.Identity on its owner."""
    norms = causal_group_norms(vae)
    if not norms:
        raise ValueError("no CausalGroupNorm found: pass a reference CausalVideoVAE or CausalVideoVAELossWrapper")
    sites = _norm_sites(vae)
    covered = set()
    for name, owner, act_attr, site_norms in sites:
        why = _norm_refusal(name, owner, act_attr, site_norms)
        if why is not None:
            raise ValueError(f"install_training_norms: {why}")
        covered.update(id(n) for n in site_norms)
    for name, m in norms:
        if id(m) not in covered:
            raise ValueError(f"install_training_norms: {name} is not followed by a SiLU the install knows how to fuse")
    for _, owner, act_attr, site_norms in sites:
        if _SAVED_ACT not in owner.__dict__:
            owner.__dict__[_SAVED_ACT] = getattr(owner, act_attr)     # kept off the module tree and the state_dict
            setattr(owner, act_attr, nn.Identity())
        for n in site_norms:
            n.forward = types.MethodType(_patched_norm_forward, n)
            setattr(n, _NORM_MARK, True)


def uninstall_training_norms(vae) -> None:
    for _, owner, act_attr, _ in _norm_sites(vae):
        act = owner.__dict__.pop(_SAVED_ACT, None)
        if act is not None:
            setattr(owner, act_attr, act)
    for _, m in causal_group_norms(vae):
        if m.__dict__.pop(_NORM_MARK, False):
            del m.forward
