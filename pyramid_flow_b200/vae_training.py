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

`lpips(input, target, module)` is LPIPS.forward (video_vae/modeling_lpips.py:32-45) of a reference LPIPS module, an autograd
function: ScalingLayer in fp32 torch ops, the 13 VGG16 convs on pf_causal_conv3d (kt = 1, ReLU fused), pf_maxpool2x2, and
pf_lpips_head_fwd over the five taps (dropout from the lin layers' Dropout when it is in training mode); the backward runs
pf_lpips_tap_bwd at the taps and the data-gradient convs with the ReLU select.  The output is fp32 [N, 1, 1, 1].
`install_training_lpips(model)` patches the LPIPS of a CausalVideoVAELossWrapper / LPIPSWithDiscriminator / LPIPS;
`uninstall_training_lpips` restores it.  The three installs compose in any order.
"""
from __future__ import annotations

import types
import weakref
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


# ------------------------------------------------------------------------------------------------------------------ LPIPS
# vgg16().features[:30] as LPIPS slices it (video_vae/modeling_lpips.py:67-89): (in, out) of the 13 conv3x3 + ReLU, the
# convs per slice, a MaxPool2d(2, 2) in front of slices 2-5; the five slice outputs are the taps relu1_2 ... relu5_3.
VGG16_CONVS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
               (512, 512), (512, 512), (512, 512), (512, 512))
VGG16_SLICES = (2, 2, 3, 3, 3)
_LPIPS_MARK = "_pf_training_lpips"
_lpips_filters = {}


def _frozen_layout(weight: torch.Tensor, kind: str, build):
    """A re-layout of a frozen weight, built once per (tensor, in-place version).  The entry holds a weak reference to the
    tensor, so a new tensor at a freed tensor's address is never served the old layout."""
    key = (kind, weight.device, weight.data_ptr(), tuple(weight.shape))
    hit = _lpips_filters.get(key)
    if hit is None or hit[0]() is not weight or hit[1] != weight._version:
        hit = _lpips_filters[key] = (weakref.ref(weight), weight._version, build(weight))
    return hit[2]


def _vgg_filter(weight: torch.Tensor) -> torch.Tensor:
    return _frozen_layout(weight, "fwd", lambda w: forward_filter(w.unsqueeze(2), _pad64(w.shape[0]), _pad64(w.shape[1])))


def _vgg_dgrad_filter(weight: torch.Tensor) -> torch.Tensor:
    return _frozen_layout(weight, "dgrad", lambda w: dgrad_filter(w.unsqueeze(2), _pad64(w.shape[0]), _pad64(w.shape[1])))


def _vgg_bias(bias: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return None if bias is None else _frozen_layout(bias, "bias", lambda b: b.detach().float().contiguous())


def _lin_weight(conv: nn.Conv2d) -> torch.Tensor:
    return _frozen_layout(conv.weight, "lin", lambda w: w.detach().float().reshape(-1).contiguous())


def _vgg_modules(lp: nn.Module) -> List[List[nn.Module]]:
    net = getattr(lp, "net", None)
    return [list(getattr(net, f"slice{s + 1}", nn.Sequential()).children()) for s in range(5)]


def _lin_layers(lp: nn.Module) -> List[nn.Sequential]:
    return [getattr(getattr(lp, f"lin{k}", None), "model", None) for k in range(5)]


def _lpips_refusal(lp: nn.Module) -> Optional[str]:
    trainable = [n for n, p in lp.named_parameters() if p.requires_grad]
    if trainable:
        return f"parameters {trainable[:3]} require grad (the op computes no LPIPS weight gradient)"
    sl = getattr(lp, "scaling_layer", None)
    if sl is None or getattr(sl, "shift", None) is None or sl.shift.numel() != 3 or sl.scale.numel() != 3:
        return "no ScalingLayer with 3-channel shift / scale buffers"
    ci = 0
    for s, mods in enumerate(_vgg_modules(lp)):
        want = 2 * VGG16_SLICES[s] + (s > 0)
        if len(mods) != want:
            return f"net.slice{s + 1} has {len(mods)} modules, not the {want} of vgg16().features"
        if s > 0:
            pool = mods[0]
            if not (type(pool) is nn.MaxPool2d and pool.kernel_size in (2, (2, 2)) and pool.stride in (2, (2, 2))
                    and pool.padding in (0, (0, 0)) and pool.dilation in (1, (1, 1)) and not pool.ceil_mode):
                return f"net.slice{s + 1}: {pool} is not MaxPool2d(2, 2)"
        for conv, act in zip(mods[s > 0::2], mods[1 + (s > 0)::2]):
            if not (type(conv) is nn.Conv2d and tuple(conv.kernel_size) == (3, 3) and tuple(conv.stride) == (1, 1)
                    and tuple(conv.padding) == (1, 1) and tuple(conv.dilation) == (1, 1) and conv.groups == 1
                    and conv.padding_mode == "zeros"):
                return f"net.slice{s + 1}: {conv} is not a 3x3 / pad 1 / stride 1 Conv2d"
            if (conv.in_channels, conv.out_channels) != VGG16_CONVS[ci]:
                return f"net.slice{s + 1}: {conv} is not VGG16's conv {ci} {VGG16_CONVS[ci]}"
            if type(act) is not nn.ReLU:
                return f"net.slice{s + 1}: {act} after a conv is not nn.ReLU"
            ci += 1
    taps_c = (64, 128, 256, 512, 512)
    for k, model in enumerate(_lin_layers(lp)):
        mods = list(model.children()) if isinstance(model, nn.Sequential) else []
        drop = mods[0] if len(mods) == 2 and type(mods[0]) is nn.Dropout else None
        conv = mods[-1] if mods and len(mods) == 1 + (drop is not None) else None
        if not (type(conv) is nn.Conv2d and tuple(conv.kernel_size) == (1, 1) and conv.bias is None
                and conv.out_channels == 1 and conv.in_channels == taps_c[k] and conv.groups == 1):
            return f"lin{k} is not [nn.Dropout] + a bias-free 1x1 Conv2d({taps_c[k]}, 1)"
        if drop is not None and not 0.0 <= drop.p < 1.0:
            return f"lin{k}: dropout p={drop.p} is not in [0, 1)"
    return None


def _lpips_dropout(lp: nn.Module) -> float:
    """The dropout probability every lin_k applies now: its Dropout's p in training mode, 0 in eval mode."""
    ps = set()
    for model in _lin_layers(lp):
        drop = model[0] if type(model[0]) is nn.Dropout else None
        ps.add(float(drop.p) if drop is not None and drop.training else 0.0)
    if len(ps) != 1:
        raise ValueError(f"lpips: the lin layers apply different dropout probabilities {sorted(ps)}; the head draws one p")
    return ps.pop()


def _vgg_forward(x: torch.Tensor, lp: nn.Module, keep_all: bool):
    """ScalingLayer + the 13 convs (ReLU fused) and the pools of one branch: (the 5 taps, every ReLU output if keep_all)."""
    n, _, h, w = x.shape
    sl = lp.scaling_layer
    xs = (x.float() - sl.shift.float()) / sl.scale.float()
    a = torch.empty(n, 1, h, w, 64, device=x.device, dtype=torch.bfloat16)
    ops.conv3d_pack(xs.unsqueeze(2), a, t_offset=0)
    taps, acts = [], []
    for s, mods in enumerate(_vgg_modules(lp)):
        if s > 0:
            c = a.shape[-1]
            pooled = torch.empty(n, 1, h // 2, w // 2, c, device=x.device, dtype=torch.bfloat16)
            ops.maxpool2x2(a.view(n, h, w, c), pooled.view(n, h // 2, w // 2, c))
            a, h, w = pooled, h // 2, w // 2
        for conv in mods[s > 0::2]:
            y = torch.empty(n, 1, h, w, conv.out_channels, device=x.device, dtype=torch.bfloat16)
            ops.causal_conv3d(a, _vgg_filter(conv.weight), _vgg_bias(conv.bias), y, kernel=(1, 3, 3), relu=True)
            a = y
            if keep_all:
                acts.append(y)
        taps.append(a)
    return taps, acts


def _vgg_backward(acts, other_taps, lp, g, p, seed, x_shape, x_dtype):
    """The input gradient of one branch: the slices in reverse, the tap backward at each tap, the data-gradient convs with
    the ReLU select inside a slice, and the first conv's 3 channels in fp32, through the ScalingLayer."""
    lins = [_lin_weight(m[-1]) for m in _lin_layers(lp)]
    slices = _vgg_modules(lp)
    end, d_next = len(acts), None
    for s in reversed(range(5)):
        convs = slices[s][s > 0::2]
        mine = acts[end - len(convs):end]
        n, _, h, w, c = mine[-1].shape
        dz = torch.empty_like(mine[-1])
        ops.lpips_tap_bwd(mine[-1].view(n, h, w, c), other_taps[s].view(n, h, w, c), lins[s], g, d_next, dz.view(n, h, w, c),
                          tap=s, p=p, seed=seed)
        for j in reversed(range(len(convs))):
            wgt = _vgg_dgrad_filter(convs[j].weight)
            if j > 0:
                out = torch.empty_like(mine[j - 1])
                ops.causal_conv3d(dz, wgt, None, out, kernel=(1, 3, 3), select=mine[j - 1])
                dz = out
            elif s > 0:
                out = torch.empty(n, 1, h, w, convs[j].in_channels, device=dz.device, dtype=torch.bfloat16)
                ops.causal_conv3d(dz, wgt, None, out, kernel=(1, 3, 3))
                d_next = out.view(n, h, w, convs[j].in_channels)
            else:
                out = torch.empty(n, 1, h, w, 3, device=dz.device, dtype=torch.float32)
                ops.causal_conv3d(dz, wgt, None, out, kernel=(1, 3, 3), store_channels=3)
                dx = out.view(n, h, w, 3).permute(0, 3, 1, 2) / lp.scaling_layer.scale.float()
        end -= len(convs)
    return dx.to(x_dtype).reshape(x_shape)


class _LPIPS(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, x1, lp, p, seed):
        need = ctx.needs_input_grad[:2]
        taps0, acts0 = _vgg_forward(x0, lp, need[0])
        taps1, acts1 = _vgg_forward(x1, lp, need[1])
        val = torch.empty(x0.shape[0], device=x0.device, dtype=torch.float32)
        ops.lpips_head_fwd([t.view(t.shape[0], *t.shape[2:]) for t in taps0], [t.view(t.shape[0], *t.shape[2:]) for t in taps1],
                           [_lin_weight(m[-1]) for m in _lin_layers(lp)], val, p=p, seed=seed)
        # a branch that needs a gradient keeps every ReLU output (its taps among them), the other one its five taps;
        # through save_for_backward, so saved-tensor hooks manage them
        kept0 = acts0 if need[0] else taps0
        kept1 = acts1 if need[1] else taps1
        ctx.save_for_backward(*kept0, *kept1, *([seed] if seed is not None else []))
        ctx.lp, ctx.p, ctx.n0, ctx.n1, ctx.has_seed = lp, p, len(kept0), len(kept1), seed is not None
        ctx.shapes, ctx.dtypes = (x0.shape, x1.shape), (x0.dtype, x1.dtype)
        return val.view(-1, 1, 1, 1)

    @staticmethod
    def backward(ctx, gval):
        saved = ctx.saved_tensors
        kept = (saved[:ctx.n0], saved[ctx.n0:ctx.n0 + ctx.n1])
        seed = saved[-1] if ctx.has_seed else None
        tap_at = [sum(VGG16_SLICES[:s + 1]) - 1 for s in range(5)]
        taps = [k if len(k) == 5 else [k[i] for i in tap_at] for k in kept]
        g = gval.reshape(-1).float().contiguous()
        grads = [None, None]
        for b in (0, 1):
            if ctx.needs_input_grad[b]:
                grads[b] = _vgg_backward(kept[b], taps[1 - b], ctx.lp, g, ctx.p, seed, ctx.shapes[b], ctx.dtypes[b])
        return grads[0], grads[1], None, None, None


def lpips(input: torch.Tensor, target: torch.Tensor, module: nn.Module) -> torch.Tensor:
    """LPIPS.forward(input, target) (video_vae/modeling_lpips.py:32-45) of the reference LPIPS `module` on the library's
    kernels: fp32 [N, 1, 1, 1].  input / target: [N, 3, H, W] bf16 or fp32, H and W multiples of 16; gradients flow to
    either or both, in each one's dtype.  The lin layers' Dropout applies when the module is in training mode (p from the
    module, the mask from torch's CUDA generator: torch.manual_seed reproduces it)."""
    why = _lpips_refusal(module)
    if why is not None:
        raise ValueError(f"lpips: {why}")
    if input.dim() != 4 or input.shape != target.shape or input.shape[1] != 3:
        raise ValueError(f"lpips: input {tuple(input.shape)} and target {tuple(target.shape)} are not one [N, 3, H, W] shape")
    if input.shape[2] % 16 or input.shape[3] % 16:
        raise ValueError(f"lpips: H and W must be multiples of 16 (four 2x2 max-pools), got {tuple(input.shape[2:])}")
    for t in (input, target):
        if t.dtype not in (torch.bfloat16, torch.float32):
            raise TypeError(f"lpips: inputs must be bf16 or fp32, got {t.dtype}")
    if not (input.is_cuda and target.is_cuda):
        raise RuntimeError("lpips runs on the library's CUDA kernels: input and target must be CUDA tensors (there is no "
                           "CPU path)")
    _require_device_once()
    p = _lpips_dropout(module)
    seed = torch.empty(1, device=input.device, dtype=torch.int64).random_() if p > 0 else None
    return _LPIPS.apply(input, target, module, p, seed)


def _patched_lpips_forward(self, input, target):
    return lpips(input, target, self)


def _lpips_module(obj: nn.Module) -> nn.Module:
    """The LPIPS of a CausalVideoVAELossWrapper (.loss.perceptual_loss), an LPIPSWithDiscriminator or an LPIPS."""
    loss = getattr(obj, "loss", None)
    if isinstance(loss, nn.Module):
        obj = loss
    inner = getattr(obj, "perceptual_loss", None)
    if isinstance(inner, nn.Module):
        obj = inner
    if type(obj).__name__ != "LPIPS":
        raise ValueError("no LPIPS found: pass a reference CausalVideoVAELossWrapper, LPIPSWithDiscriminator or LPIPS")
    return obj


def install_training_lpips(model) -> None:
    """Run the reference LPIPS of `model` (see _lpips_module) on `lpips`."""
    lp = _lpips_module(model)
    why = _lpips_refusal(lp)
    if why is not None:
        raise ValueError(f"install_training_lpips: {why}")
    lp.forward = types.MethodType(_patched_lpips_forward, lp)
    setattr(lp, _LPIPS_MARK, True)


def uninstall_training_lpips(model) -> None:
    lp = _lpips_module(model)
    if lp.__dict__.pop(_LPIPS_MARK, False):
        del lp.forward
