"""ctypes binding of the C ABI in ``include/sfb200.h`` (libsfb200.so).

There is no fallback: if the shared library is missing, or an entry point fails, an exception is
raised.  The library is built in-tree by ``__graft_entry__.build()`` / ``csrc/Makefile``.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SFB_LIB_PATH: A/B builds of the same ABI (experiments only; still no fallback)
LIB_PATH = os.environ.get("SFB_LIB_PATH") or os.path.join(_HERE, "libsfb200.so")

ABI_VERSION = 4  # SFB_ABI_VERSION of include/sfb200.h
SFB_F16, SFB_BF16, SFB_F32 = 0, 1, 2
LORA_MAX_ADAPTERS, LORA_MAX_RANK = 8, 256
A_MATRIX, A_CONV3X3, A_UPCONV2X, A_CONV3X1, A_CONV3X3_GN, A_DOWNCONV3X3 = 0, 1, 2, 3, 4, 5
ROW_IDX_DIV_MOD, ROW_IDX_TEMPORAL_CTX = 0, 1
EPI_STORE, EPI_GEGLU, EPI_QKV, EPI_STORE_F32 = 0, 1, 2, 3
ACT_NONE, ACT_QUICK_GELU, ACT_GELU, ACT_SILU, ACT_RELU = 0, 1, 2, 3, 4
XFORM_NONE, XFORM_TANH3, XFORM_UNIT = 0, 1, 2
C64_SAME, C64_STRIDE2, C64_UP2X = 0, 1, 2


class GemmParams(C.Structure):
    _fields_ = [
        ("tmap_a", C.c_void_p), ("tmap_b", C.c_void_p),
        ("a_mode", C.c_int32), ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("dtype", C.c_int32),
        ("img_n", C.c_int32), ("img_h", C.c_int32), ("img_w", C.c_int32), ("cin", C.c_int32),
        ("conv_stride", C.c_int32), ("box_h", C.c_int32), ("box_n", C.c_int32),
        ("box_w", C.c_int32),
        ("splits", C.c_int32), ("ws", C.c_void_p), ("defer_finish", C.c_int32),
        ("epi", C.c_int32), ("out", C.c_void_p), ("ldo", C.c_int32),
        ("bias", C.c_void_p), ("rowbias", C.c_void_p),
        ("rows_per_img", C.c_int32), ("ld_rowbias", C.c_int32),
        ("residual", C.c_void_p), ("ldr", C.c_int32), ("geglu_n_out", C.c_int32),
        ("q", C.c_void_p), ("k", C.c_void_p), ("vt", C.c_void_p),
        ("heads", C.c_int32), ("head_dim", C.c_int32), ("which_base", C.c_int32),
        ("seq", C.c_int32), ("q_pitch", C.c_int32), ("q_rows", C.c_int32),
        ("k_rows", C.c_int32), ("vt_rows", C.c_int32), ("vt_pitch", C.c_int32),
        ("cta_pair", C.c_int32), ("persistent", C.c_int32), ("b_plain", C.c_int32),
        ("rowstats_out", C.c_void_p), ("ln_rowstats", C.c_void_p), ("ln_colsum", C.c_void_p),
        ("ln_eps", C.c_float), ("ln_dim", C.c_int32), ("act", C.c_int32),
        ("rowstats_out_slots", C.c_int32), ("ln_slots", C.c_int32),
        ("gn_scale_shift", C.c_void_p), ("gn_silu", C.c_int32),
    ]


class AttnParams(C.Structure):
    _fields_ = [
        ("tmap_q", C.c_void_p), ("tmap_k", C.c_void_p), ("tmap_vt", C.c_void_p),
        ("out", C.c_void_p),
        ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
        ("seq_q", C.c_int32), ("seq_kv", C.c_int32),
        ("q_rows", C.c_int32), ("k_rows", C.c_int32), ("vt_rows", C.c_int32),
        ("dtype", C.c_int32), ("scale", C.c_float), ("kv_tile", C.c_int32), ("causal", C.c_int32),
    ]


class AttnIpParams(C.Structure):
    _fields_ = [
        ("base", AttnParams), ("tmap_k_ip", C.c_void_p), ("tmap_vt_ip", C.c_void_p),
        ("seq_ip", C.c_int32), ("k_ip_rows", C.c_int32), ("ip_scale", C.c_void_p),
    ]


class GnParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("y", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("stats", C.c_void_p),
        ("n", C.c_int32), ("hw", C.c_int32), ("c", C.c_int32), ("ldx", C.c_int32),
        ("ldy", C.c_int32), ("groups", C.c_int32),
        ("eps", C.c_float), ("silu", C.c_int32), ("dtype", C.c_int32),
        ("sync_counter", C.c_void_p),
        ("part_ws", C.c_void_p), ("part_splits", C.c_int32), ("part_c", C.c_int32),
        ("part_ld", C.c_int32), ("part_bias", C.c_void_p), ("part_rowbias", C.c_void_p),
        ("part_ld_rowbias", C.c_int32), ("part_residual", C.c_void_p), ("part_ldr", C.c_int32),
    ]


class LnParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("y", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("rows", C.c_int32), ("c", C.c_int32), ("ldx", C.c_int32), ("ldy", C.c_int32),
        ("eps", C.c_float), ("dtype", C.c_int32),
    ]


class SmallLinearParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("add16", C.c_void_p),
        ("y16", C.c_void_p), ("y32", C.c_void_p),
        ("batch", C.c_int32), ("n", C.c_int32), ("k", C.c_int32), ("ldx", C.c_int32),
        ("ldy", C.c_int32), ("act_in", C.c_int32), ("act_out", C.c_int32), ("dtype", C.c_int32),
    ]


class TemporalAttnParams(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("out", C.c_void_p),
                ("batch", C.c_int32), ("frames", C.c_int32), ("seq", C.c_int32), ("heads", C.c_int32),
                ("head_dim", C.c_int32), ("ld_qkv", C.c_int32), ("ld_out", C.c_int32), ("dtype", C.c_int32),
                ("scale", C.c_float)]


class FrameAttnParams(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("frame_bias", C.c_void_p), ("out", C.c_void_p),
                ("batch", C.c_int32), ("frames", C.c_int32), ("seq", C.c_int32), ("heads", C.c_int32),
                ("head_dim", C.c_int32), ("ld_qkv", C.c_int32), ("ld_bias", C.c_int32), ("ld_out", C.c_int32),
                ("dtype", C.c_int32), ("scale", C.c_float)]


class RowOpParams(C.Structure):
    _fields_ = [("x", C.c_void_p), ("x2", C.c_void_p), ("vec", C.c_void_p), ("y", C.c_void_p),
                ("rowstats_out", C.c_void_p), ("mix_factor", C.c_void_p),
                ("rows", C.c_int32), ("c", C.c_int32), ("ldx", C.c_int32), ("ldx2", C.c_int32),
                ("ldv", C.c_int32), ("ldy", C.c_int32), ("dtype", C.c_int32),
                ("mode", C.c_int32), ("div", C.c_int32), ("mod", C.c_int32), ("frames", C.c_int32),
                ("seq", C.c_int32), ("batch", C.c_int32), ("rowstats_slots", C.c_int32)]


class AddNchwItem(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("n", C.c_int32), ("c", C.c_int32),
                ("hw", C.c_int32), ("ld_dst", C.c_int32)]


class AddNchwParams(C.Structure):
    _fields_ = [("count", C.c_int32), ("dtype", C.c_int32), ("items", AddNchwItem * 16)]


class ConvSmallParams(C.Structure):
    _fields_ = [("x", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p), ("y", C.c_void_p),
                ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("cin", C.c_int32), ("cout", C.c_int32),
                ("stride", C.c_int32), ("ldx", C.c_int32), ("ldy", C.c_int32), ("x_nchw", C.c_int32),
                ("silu", C.c_int32), ("dtype", C.c_int32)]


class ConvSmallExParams(C.Structure):
    _fields_ = [("base", ConvSmallParams), ("in_xform", C.c_int32), ("relu", C.c_int32)]


class ConvC64Params(C.Structure):
    _fields_ = [("x", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p), ("residual", C.c_void_p),
                ("y", C.c_void_p), ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("ldx", C.c_int32),
                ("ldy", C.c_int32), ("ldr", C.c_int32), ("mode", C.c_int32), ("relu", C.c_int32),
                ("dtype", C.c_int32)]


class NchwScaledItem(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("n", C.c_int32), ("c", C.c_int32),
                ("hw", C.c_int32), ("ld_src", C.c_int32)]


class NhwcToNchwParams(C.Structure):
    _fields_ = [("count", C.c_int32), ("dtype", C.c_int32), ("scale", C.c_void_p), ("items", NchwScaledItem * 16)]


class FreeUParams(C.Structure):
    _fields_ = [("x", C.c_void_p), ("bs", C.c_void_p), ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
                ("c_hidden", C.c_int32), ("c_skip", C.c_int32), ("ld", C.c_int32), ("dtype", C.c_int32)]


class LoraAdapter(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("rank", C.c_int32), ("lda", C.c_int32), ("ldb", C.c_int32),
                ("a_dtype", C.c_int32), ("b_dtype", C.c_int32), ("scale", C.c_float)]


class LoraMergeParams(C.Structure):
    _fields_ = [("w", C.c_void_p), ("out", C.c_void_p), ("n", C.c_int32), ("k", C.c_int32), ("ldw", C.c_int32),
                ("ldo", C.c_int32), ("w_dtype", C.c_int32), ("out_dtype", C.c_int32), ("count", C.c_int32),
                ("adapters", LoraAdapter * LORA_MAX_ADAPTERS)]


# every symbol include/sfb200.h declares: (name, restype, argtypes)
_I32, _U32, _U64, _VP, _F = C.c_int32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_float
SYMBOLS = {
    "sfb_abi_version": (C.c_int, []),
    "sfb_last_error": (C.c_char_p, []),
    "sfb_launch_count": (C.c_uint64, []),
    "sfb_set_pdl": (None, [C.c_int]),
    "sfb_sm_count": (C.c_int, []),
    "sfb_tmap_2d": (C.c_int, [_VP, _VP, _U64, _U64, _U64, _U32]),
    "sfb_tmap_nhwc": (C.c_int, [_VP, _VP, _U32, _U32, _U32, _U32, _U64, _U32, _U32, _U32, _U32]),
    "sfb_gemm": (C.c_int, [C.POINTER(GemmParams), _VP]),
    "sfb_attention": (C.c_int, [C.POINTER(AttnParams), _VP]),
    "sfb_attention_ip": (C.c_int, [C.POINTER(AttnIpParams), _VP]),
    "sfb_group_norm_stats": (C.c_int, [C.POINTER(GnParams), _VP]),
    "sfb_group_norm_apply": (C.c_int, [C.POINTER(GnParams), _VP]),
    "sfb_group_norm_scale_shift": (C.c_int, [C.POINTER(GnParams), _VP, _VP]),
    "sfb_group_norm_fused_fits": (C.c_int, [C.POINTER(GnParams)]),
    "sfb_group_norm_ws_floats": (C.c_int, [_I32, _I32]),
    "sfb_group_norm_fused": (C.c_int, [C.POINTER(GnParams), _VP]),
    "sfb_layer_norm": (C.c_int, [C.POINTER(LnParams), _VP]),
    "sfb_timestep_embed": (C.c_int, [_VP, _I32, _I32, _I32, _F, _VP, _I32, _I32, _VP]),
    "sfb_small_linear": (C.c_int, [C.POINTER(SmallLinearParams), _VP]),
    "sfb_im2col_in": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _VP]),
    "sfb_im2col_in_wide": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _VP]),
    "sfb_conv_in": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_conv_out": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_conv_out_temporal": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _I32,
                                        _I32, _VP]),
    "sfb_upsample2x": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_temporal_attention": (C.c_int, [C.POINTER(TemporalAttnParams), _VP]),
    "sfb_frame_attention": (C.c_int, [C.POINTER(FrameAttnParams), _VP]),
    "sfb_row_broadcast_add": (C.c_int, [C.POINTER(RowOpParams), _VP]),
    "sfb_alpha_blend": (C.c_int, [C.POINTER(RowOpParams), _VP]),
    "sfb_add_nchw_residuals": (C.c_int, [C.POINTER(AddNchwParams), _VP]),
    "sfb_copy2d": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _VP]),
    "sfb_row_softmax": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_pointwise_nchw": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_memset": (C.c_int, [_VP, _I32, C.c_size_t, _VP]),
    "sfb_embed_tokens": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_rowstats_slots": (C.c_int, [_I32]),
    "sfb_clip_pool": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_patchify": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_conv3x3_small": (C.c_int, [C.POINTER(ConvSmallParams), _VP]),
    "sfb_conv3x3_small_ex": (C.c_int, [C.POINTER(ConvSmallExParams), _VP]),
    "sfb_conv3x3_c64": (C.c_int, [C.POINTER(ConvC64Params), _VP]),
    "sfb_nhwc_to_nchw_scaled": (C.c_int, [C.POINTER(NhwcToNchwParams), _VP]),
    "sfb_lora_merge": (C.c_int, [C.POINTER(LoraMergeParams), _VP]),
    "sfb_pixel_unshuffle": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_avg_pool2x2": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "sfb_freeu": (C.c_int, [C.POINTER(FreeUParams), _VP]),
}

_lib = None


class SfbError(RuntimeError):
    pass


def lib():
    """Load libsfb200.so (once).  Raises if the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SfbError(
                f"{LIB_PATH} not found: the sm_90a CUDA extension is not built "
                "(run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C "
                "stable-fast_b200/csrc`).  There is no CPU fallback.")
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        if h.sfb_abi_version() != ABI_VERSION:
            raise SfbError("libsfb200.so ABI version mismatch")
        _lib = h
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().sfb_last_error().decode("utf-8", "replace")
        raise SfbError(f"{what or 'sfb call'} failed ({rc}): {msg}")


class TensorMap:
    """Owns one 128-byte CUtensorMap in 64-byte-aligned host memory."""

    def __init__(self):
        self._buf = (C.c_uint8 * 256)()
        base = C.addressof(self._buf)
        self.ptr = (base + 63) & ~63

    @classmethod
    def matrix(cls, base_ptr, rows, cols, pitch, box_rows):
        t = cls()
        check(lib().sfb_tmap_2d(t.ptr, base_ptr, rows, cols, pitch, box_rows), "sfb_tmap_2d")
        return t

    @classmethod
    def nhwc(cls, base_ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride=1):
        t = cls()
        check(lib().sfb_tmap_nhwc(t.ptr, base_ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride),
              "sfb_tmap_nhwc")
        return t
