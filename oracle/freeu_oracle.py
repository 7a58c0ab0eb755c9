"""ORACLE (test infrastructure, NOT product code): FreeU (Si et al., "FreeU: Free Lunch in Diffusion U-Net") as
diffusers computes it, on an ``oracle.unet_oracle`` UNet.

Restates diffusers' ``utils.torch_utils.fourier_filter`` and ``apply_freeu``, the FreeU branch of
``UpBlock2D.forward`` / ``CrossAttnUpBlock2D.forward`` (up block i has ``resolution_idx = i``; a block applies FreeU
only when all four of its own ``s1, s2, b1, b2`` are truthy), and ``UNet2DConditionModel.enable_freeu`` /
``disable_freeu``.  ``enable_freeu(unet, ...)`` sets the four attributes on every up block, as diffusers does, and
gives each up block of the oracle UNet diffusers' FreeU-aware forward; with FreeU off that forward computes exactly
``unet_oracle.UpBlock.forward``.  ``t2i_adapter_oracle.unet_forward`` (and the UNet's own forward) reach it through
``blk(...)``.  Only ``tests/`` may import this module.
"""
import types

import torch

FREEU_KEYS = ("s1", "s2", "b1", "b2")


def fourier_filter(x_in: torch.Tensor, threshold: int, scale: float) -> torch.Tensor:
    """diffusers ``fourier_filter``: scale the centre box of half-width `threshold` of the fftshift-ed 2-D spectrum of
    every (image, channel) by `scale` (an fp32 mask, as in diffusers).  The FFT runs in the input dtype at
    power-of-two sizes (cuFFT's half precision for fp16) except for bf16, else in fp32."""
    x = x_in
    B, C, H, W = x.shape
    if (W & (W - 1)) != 0 or (H & (H - 1)) != 0:
        x = x.to(dtype=torch.float32)
    elif x.dtype == torch.bfloat16:
        x = x.to(dtype=torch.float32)
    x_freq = torch.fft.fftn(x, dim=(-2, -1))
    x_freq = torch.fft.fftshift(x_freq, dim=(-2, -1))
    B, C, H, W = x_freq.shape
    mask = torch.ones((B, C, H, W), device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    x_freq = x_freq * mask
    x_freq = torch.fft.ifftshift(x_freq, dim=(-2, -1))
    x_filtered = torch.fft.ifftn(x_freq, dim=(-2, -1)).real
    return x_filtered.to(dtype=x_in.dtype)


def apply_freeu(resolution_idx, hidden_states, res_hidden_states, **freeu_kwargs):
    """diffusers ``apply_freeu``: up block 0 (1) scales the first half of the backbone channels by b1 (b2), in place,
    and filters the skip tensor with s1 (s2); later blocks are left alone."""
    for idx, (b, s) in enumerate((("b1", "s1"), ("b2", "s2"))):
        if resolution_idx == idx:
            num_half_channels = hidden_states.shape[1] // 2
            hidden_states[:, :num_half_channels] = hidden_states[:, :num_half_channels] * freeu_kwargs[b]
            res_hidden_states = fourier_filter(res_hidden_states, threshold=1, scale=freeu_kwargs[s])
    return hidden_states, res_hidden_states


def _up_block_forward(self, x, skips, temb, ctx):
    """``unet_oracle.UpBlock.forward`` with diffusers' FreeU branch in front of each resnet's concatenation."""
    for i, r in enumerate(self.resnets):
        skip = skips.pop()
        if all(getattr(self, k, None) for k in FREEU_KEYS):
            x, skip = apply_freeu(self.resolution_idx, x, skip, s1=self.s1, s2=self.s2, b1=self.b1, b2=self.b2)
        x = torch.cat([x, skip], dim=1)
        x = r(x, temb)
        if self.attentions is not None:
            x = self.attentions[i](x, ctx)
    if self.upsamplers is not None:
        x = self.upsamplers[0](x)
    return x


def _install(unet):
    for i, blk in enumerate(unet.up_blocks):
        blk.resolution_idx = i
        blk.forward = types.MethodType(_up_block_forward, blk)


def enable_freeu(unet, s1, s2, b1, b2):
    """diffusers ``UNet2DConditionModel.enable_freeu``: the four FreeU values on every up block."""
    _install(unet)
    for blk in unet.up_blocks:
        blk.s1, blk.s2, blk.b1, blk.b2 = s1, s2, b1, b2


def disable_freeu(unet):
    """diffusers ``UNet2DConditionModel.disable_freeu``: every up block's FreeU values set to None."""
    _install(unet)
    for blk in unet.up_blocks:
        for k in FREEU_KEYS:
            if hasattr(blk, k) or getattr(blk, k, None) is not None:
                setattr(blk, k, None)
