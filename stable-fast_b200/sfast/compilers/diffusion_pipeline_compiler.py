"""``sfast.compilers.diffusion_pipeline_compiler`` -- same names, fields and call convention as
/root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:20-190, with the UNet hot path
executed by the H100-native runtime (``sfast_b200``).

    from sfast.compilers.diffusion_pipeline_compiler import compile, CompilationConfig
    config = CompilationConfig.Default()
    config.enable_cuda_graph = True
    pipe = compile(pipe, config)          # same pipeline object, unet.forward replaced

Field mapping (all 11 reference fields are accepted):
  enable_cuda_graph      -> capture the whole UNet step as one CUDA graph per (B, H, W, dtype)
  enable_jit, enable_jit_freeze, enable_cnn_optimization, enable_fused_linear_geglu,
  prefer_lowp_gemm, enable_xformers, enable_triton, memory_format
                         -> accepted; they select nothing: the native path always runs NHWC with
                            every fusion on (fp32 accumulation, erf-GELU)
  preserve_parameters    -> True (default): in-place parameter updates (LoRA switch, reference
                            README.md:228-265) and PEFT LoRA adapter changes are picked up by the next
                            call -- the packed copies are refreshed in place;
                            False: weights and adapter state are frozen at first call (``rebind()``
                            refreshes)
  trace_scheduler        -> accepted, no-op (scheduler is outside the hot path)
"""
import logging
from dataclasses import dataclass

import torch

from sfast.utils import gpu_device

logger = logging.getLogger()


class CompilationConfig:

    @dataclass
    class Default:
        memory_format: torch.memory_format = (
            torch.channels_last if gpu_device.device_has_tensor_core() else
            torch.contiguous_format)
        enable_jit: bool = True
        enable_jit_freeze: bool = True
        preserve_parameters: bool = True
        enable_cnn_optimization: bool = gpu_device.device_has_tensor_core()
        enable_fused_linear_geglu: bool = gpu_device.device_has_capability(8, 0)
        prefer_lowp_gemm: bool = True
        enable_xformers: bool = False
        enable_cuda_graph: bool = False
        enable_triton: bool = False
        trace_scheduler: bool = False


def compile(m, config):
    """Compile a diffusers pipeline in place and return it (reference `compile`, :81-124): the UNet, the
    ControlNet (``pipe.controlnet``: a ControlNetModel, or each net of a MultiControlNetModel), the VAE, the
    text encoders and the image encoder run on the native path; a ControlNet class or config the native
    path does not cover stays eager with a warning.  The T2I-Adapter (``pipe.adapter`` of the adapter pipelines: a
    T2IAdapter, or each adapter of a MultiAdapter) runs natively too, see `compile_adapter`, and the UNet adds its
    residuals (``down_intrablock_additional_residuals``) inside its step.  A loaded IP-Adapter (one plain ``ImageProjection`` or one
    IP-Adapter Plus ``IPAdapterPlusImageProjection``) runs inside the UNet's step, see `compile_unet`.  PEFT LoRA
    adapters on the UNet and the text encoders are merged into their packed weights (see `compile_unet`); adapters
    on the ControlNet, the VAE or the vision tower raise ``NotImplementedError`` at their first call.  An AnimateDiff
    pipeline's ``UNetMotionModel`` runs natively with its motion modules (see `compile_unet`); a
    ``SparseControlNetModel`` stays eager and its residuals reach the native UNet like any ControlNet's."""
    m.unet = compile_unet(m.unet, config)
    if getattr(m, 'controlnet', None) is not None:
        m.controlnet = compile_controlnet(m.controlnet, config)
    if getattr(m, 'adapter', None) is not None:
        m.adapter = compile_adapter(m.adapter, config)
    if getattr(m, 'vae', None) is not None:
        m.vae = compile_vae(m.vae, config)
    # text encoders (reference :93-112: lazy trace + CUDA graph of text_encoder / text_encoder_2)
    for attr in ('text_encoder', 'text_encoder_2'):
        if getattr(m, attr, None) is not None:
            setattr(m, attr, compile_text_encoder(getattr(m, attr), config))
    # SVD's CLIP vision tower (reference :100-103)
    if getattr(m, 'image_encoder', None) is not None:
        m.image_encoder = compile_image_encoder(m.image_encoder, config)
    if getattr(config, 'trace_scheduler', False):
        logger.warning('sfast (H100 build): trace_scheduler is ignored (scheduler.step stays eager)')
    return m


def compile_image_encoder(m, config):
    """Replace ``m.forward`` of a transformers CLIPVisionModel / CLIPVisionModelWithProjection (the SVD
    pipeline's image_encoder, reference :100-103) with the H100-native tower; anything else is returned
    unchanged with a warning."""
    from sfast_b200.runtime import compile_image_encoder_module, require_sm90
    cfg = getattr(m, 'config', None)
    if cfg is None or not hasattr(m, 'vision_model') or getattr(cfg, 'model_type', 'clip_vision_model') != 'clip_vision_model':
        logger.warning('sfast (H100 build): %s is not a CLIP vision model; left on its eager path', type(m).__name__)
        return m
    device = m.device if hasattr(m, 'device') else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    require_sm90(torch.device(device))
    return compile_image_encoder_module(m, enable_cuda_graph=bool(config.enable_cuda_graph))


def compile_text_encoder(m, config):
    """Replace ``m.forward`` of a transformers CLIPTextModel / CLIPTextModelWithProjection with the
    H100-native encoder (reference :93-112).  Any other encoder class, or one on a non-sm_90
    device, is returned unchanged with a warning."""
    from sfast_b200.runtime import compile_text_encoder_module, require_sm90
    cfg = getattr(m, 'config', None)
    if cfg is None or not hasattr(m, 'text_model') or getattr(cfg, 'model_type', 'clip_text_model') != 'clip_text_model':
        logger.warning('sfast (H100 build): %s is not a CLIP text model; left on its eager path', type(m).__name__)
        return m
    device = m.device if hasattr(m, 'device') else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    require_sm90(torch.device(device))
    return compile_text_encoder_module(m, enable_cuda_graph=bool(config.enable_cuda_graph))


def compile_controlnet(m, config):
    """Replace ``m.forward`` of a diffusers ControlNetModel with the H100-native ControlNet (the reference
    compiles it like the UNet, :89-90).  A MultiControlNetModel (one with ``.nets``) gets each net's
    forward replaced.  Any other class, or a config the native path does not cover, is left on its eager
    path with a warning."""
    nets = getattr(m, 'nets', None)
    if nets is not None:
        for net in nets:
            _compile_controlnet_net(net, config)
        return m
    return _compile_controlnet_net(m, config)


def compile_adapter(m, config):
    """Replace ``m.forward`` of a diffusers T2IAdapter ("full_adapter" or "full_adapter_xl") with the H100-native
    adapter: one plan and CUDA graph per (batch, image size, dtype); the features are fresh NCHW tensors.  A
    MultiAdapter (one with ``.adapters``) gets each adapter's forward replaced and keeps its own weighted sum.  Any
    other class, or a config the native path does not cover (``light_adapter``, channel counts that are not
    multiples of 64), is left on its eager path with a warning.  The module object is kept, so
    ``downscale_factor`` and ``total_downscale_factor`` still work."""
    adapters = getattr(m, 'adapters', None)
    if adapters is not None:
        for a in adapters:
            _compile_adapter_net(a, config)
        return m
    return _compile_adapter_net(m, config)


def _compile_adapter_net(m, config):
    from sfast_b200.runtime import compile_adapter_module, require_sm90
    from sfast_b200.t2i_adapter_plan import t2i_adapter_spec_from_config
    if type(m).__name__ != 'T2IAdapter' or not hasattr(m, 'config'):
        logger.warning('sfast (H100 build): %s is not a T2IAdapter; left on its eager path', type(m).__name__)
        return m
    try:
        t2i_adapter_spec_from_config(m.config)
    except NotImplementedError as exc:
        logger.warning('sfast (H100 build): T2I-Adapter left on its eager path (%s)', exc)
        return m
    device = m.device if hasattr(m, 'device') else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    require_sm90(torch.device(device))
    return compile_adapter_module(m, enable_cuda_graph=bool(config.enable_cuda_graph),
                                  preserve_parameters=bool(getattr(config, 'preserve_parameters', True)))


def _compile_controlnet_net(m, config):
    from sfast_b200.runtime import compile_controlnet_module, require_sm90
    from sfast_b200.unet_spec import controlnet_spec_from_config
    if type(m).__name__ != 'ControlNetModel' or not hasattr(m, 'config'):
        logger.warning('sfast (H100 build): %s is not a ControlNetModel; left on its eager path', type(m).__name__)
        return m
    try:
        controlnet_spec_from_config(m.config)
    except NotImplementedError as exc:
        logger.warning('sfast (H100 build): ControlNet left on its eager path (%s)', exc)
        return m
    device = m.device if hasattr(m, 'device') else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    require_sm90(torch.device(device))
    return compile_controlnet_module(m, enable_cuda_graph=bool(config.enable_cuda_graph),
                                     preserve_parameters=bool(getattr(config, 'preserve_parameters', True)))


def compile_unet(m, config):
    """Replace ``m.forward`` with the H100-native UNet step (reference `compile_unet`, :127-151).

    There is no CPU / eager fallback: the module must live on an sm_90 CUDA device.  A loaded IP-Adapter is
    compiled with it: a plain adapter's image projection, or IP-Adapter Plus's Resampler (its perceiver blocks
    over the image features of ``added_cond_kwargs["image_embeds"]``, ``[B, n_img, S_img, D_img]``), runs on
    the step's side stream inside the same CUDA graph, and every cross-attention adds the image-token term.
    FaceID projections, several adapters and ``ip_adapter_masks`` raise ``NotImplementedError`` by name.

    T2I-Adapter residuals (``down_intrablock_additional_residuals``, or diffusers' deprecated form: down residuals
    without a mid residual) are added where diffusers adds them, one in-place add per insertion point right after
    the tensor's producer, before any ControlNet residual; a wrong shape raises ``ValueError`` naming the index.
    Unlike diffusers, the caller's list is not consumed (diffusers pops from it).  Each number of residuals used
    gets its own plan and CUDA graph; a call without them runs the launch list of a plain step.

    PEFT LoRA adapters (diffusers' ``load_lora_weights``), loaded before or after this call, fused or not, are
    merged into the packed weights whenever the adapter state changes (``set_adapters``, ``fuse_lora``,
    ``disable_lora``, ``delete_adapters``, ...); ``cross_attention_kwargs={"scale": s}`` scales the active
    adapters for that call.  The step's launch list and CUDA graph are those of the adapter-free UNet.  DoRA,
    ``lora_bias`` and non-LoRA PEFT adapters raise ``NotImplementedError`` naming the layer.

    FreeU (``pipe.enable_freeu(s1, s2, b1, b2)`` / ``unet.enable_freeu``) is read from ``up_blocks[0]`` and
    ``[1]`` on every call, with diffusers' rule per block (on when all four of its values are truthy): the
    backbone scaling and the Fourier skip filter run natively in front of each resnet of those blocks, inside the
    CUDA graph.  Each on/off pair gets its own plan; changing the values reuses it, and with FreeU off the step
    is the plain one.

    AnimateDiff's ``UNetMotionModel`` (``forward(sample [B, C, F, H, W], timestep, encoder_hidden_states, ...)``)
    runs as B*F images with the motion modules inside the same step: the video GroupNorm, proj_in, the two
    self-attentions across the frames (with the sinusoidal position embedding) and the GEGLU FeedForward of each
    block, and proj_out.  One plan and CUDA graph per (B, F, H, W, dtype, ControlNet or not); ``timestep_cond``
    (AnimateLCM) and SDXL's ``added_cond_kwargs`` are repeated per frame, ControlNet residuals are ``[B*F, C, h,
    w]``, and PEFT LoRA adapters, motion LoRAs included, are merged as above.  ``attention_mask``, an IP-Adapter,
    FreeU, T2I-Adapter residuals, FreeNoise and more frames than ``motion_max_seq_length`` raise
    ``NotImplementedError`` by name on the call that uses them."""
    from sfast_b200.runtime import compile_unet_module, require_sm90
    device = m.device if hasattr(m, 'device') else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    require_sm90(torch.device(device))
    return compile_unet_module(m, enable_cuda_graph=bool(config.enable_cuda_graph),
                               preserve_parameters=bool(getattr(config, 'preserve_parameters', True)))


def compile_vae(m, config):
    """Replace ``m.decode`` and ``m.encode`` with the H100-native VAE decoder and encoder (reference
    `compile_vae`, :154-190, which wraps the sub-modules in auto-trace hooks).  Both share one packed
    copy of the weights.  `encode` is replaced only where the module has one (img2img and inpainting
    call it every time).  SVD's AutoencoderKLTemporalDecoder (no post_quant_conv) gets the native
    ``decode(z, num_frames, return_dict=True)``: z holds z.shape[0] / num_frames videos, one launch
    plan and CUDA graph per (frames, num_frames, latent size, dtype), so the pipeline's chunks of
    `decode_chunk_size` frames and its shorter last chunk each get their own.  Another VAE without
    post_quant_conv, or one missing any parameter of that decoder, keeps its own decode.  diffusers'
    AutoencoderTiny (TAESD / TAESDXL) gets the native ``decode(x, generator=None, return_dict=True)`` and
    ``encode(x, return_dict=True)`` (one plan and CUDA graph per (kind, batch, size, dtype); `use_slicing`
    runs the whole batch in one plan, `use_tiling` stays on the module's own methods); a tiny VAE whose
    config the native path does not compute (e.g. 16-channel latents) stays eager with a warning.  fp32 calls
    (force_upcast) and diffusers' tiled encode stay on the module's eager path.  A VAE without a `decode` method is returned unchanged
    with a warning (the reference, too, only hooks what it can trace)."""
    from sfast_b200.runtime import compile_vae_module, require_sm90
    if not hasattr(m, 'decode') or not hasattr(m, 'config'):
        logger.warning('sfast (H100 build): VAE without decode()/config is left on its eager path')
        return m
    device = m.device if hasattr(m, 'device') else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    require_sm90(torch.device(device))
    return compile_vae_module(m, enable_cuda_graph=bool(config.enable_cuda_graph))
