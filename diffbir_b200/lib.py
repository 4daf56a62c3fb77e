"""ctypes binding of libdiffbir_b200.so (the C ABI declared in include/diffbir_b200.h).

The product path fails loudly when the CUDA library is missing: there is no CPU or
PyTorch-eager fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import torch

import os

_HERE = Path(__file__).resolve().parent
# DBIR_OPERANDS=bf16 loads the -DDBIR_OPERAND_BF16 build (bf16 tensor-core operands); default fp16 operands.
_OPERANDS = os.environ.get("DBIR_OPERANDS", "fp16").lower()
if _OPERANDS not in ("fp16", "bf16"):
    raise ValueError(f"DBIR_OPERANDS={_OPERANDS!r}: expected fp16 or bf16")
LIB_PATH = _HERE / ("libdiffbir_b200_bf16.so" if _OPERANDS == "bf16" else "libdiffbir_b200.so")
_lib = None
_launches = 0  # kernels launched through this binding (bench.py reports it)


class DbirError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("b", C.c_void_p), ("out", C.c_void_p),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("residual", C.c_void_p),
        ("lda", C.c_int64), ("ldb", C.c_int64), ("ldo", C.c_int64), ("ldr", C.c_int64),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("a_mode", C.c_int32),
        ("img_n", C.c_int32), ("img_h", C.c_int32), ("img_w", C.c_int32), ("img_c", C.c_int32),
        ("ksize", C.c_int32),
        ("rows_per_vec", C.c_int32), ("out_kind", C.c_int32), ("act", C.c_int32),
        ("geglu", C.c_int32), ("force_bn", C.c_int32),
        ("alpha", C.c_float), ("act_param", C.c_float),
        ("bias_per_row", C.c_int32), ("groups", C.c_int32),
        ("splitk_ws", C.c_void_p), ("splitk_ws_bytes", C.c_int64),
        ("split_k", C.c_int32), ("cta_pair", C.c_int32),
        ("gn_partials", C.c_void_p), ("gn_rows_per_img", C.c_int32),
    ]


def load():
    """Loads the shared library (building is the job of __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise DbirError(
            f"{LIB_PATH} not found: build it with `python -m diffbir_b200.build{' --bf16' if _OPERANDS == 'bf16' else ''}` "
            "(there is no CPU fallback)")
    lib = C.CDLL(str(LIB_PATH))
    lib.dbir_last_error.restype = C.c_char_p
    lib.dbir_version.restype = C.c_char_p
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().dbir_last_error().decode(errors="replace")
        raise DbirError(f"{what} failed (rc={rc}): {msg}")


_record = None    # list of (kind, info, flops, thunk) while recording


def record_begin():
    """Records every GEMM / attention launch (arguments included) so bench.py can replay exactly the
    tensor-core kernels of one forward inside a CUDA graph and time them with CUDA events."""
    global _record
    _record = []


def record_end():
    global _record
    out, _record = _record, None
    return out


def count_launch(n: int = 1):
    global _launches
    _launches += n


def launches() -> int:
    return _launches


def operand_dtype() -> torch.dtype:
    return torch.float16 if load().dbir_operand_kind() == 1 else torch.bfloat16


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


ACT = {None: 0, "none": 0, "gelu": 1, "lrelu": 2, "silu": 3, "quick_gelu": 4}


def gemm(a, b, out, *, M, N, K, bias=None, rowvec=None, rows_per_vec=0, residual=None,
         lda=0, ldb=0, ldo=None, ldr=None, conv=None, act=None, act_param=0.0, alpha=1.0,
         geglu=False, force_bn=0, bias_per_row=False, splitk_ws=None, split_k=0, cta_pair=0,
         gn_partials=None, gn_rows_per_img=0, groups=1):
    """out = residual + alpha * act(A @ B^T + bias + rowvec). conv = (n, h, w, c, ksize).
    geglu: False / True (= 1, values * gelu(gates)) or 2 (values * silu(gates)), weights packed per force_bn tile."""
    lib = load()
    g = GemmArgs()
    g.a, g.b, g.out = a.data_ptr(), b.data_ptr(), out.data_ptr()
    g.bias, g.rowvec, g.residual = _ptr(bias), _ptr(rowvec), _ptr(residual)
    n_out = N // 2 if geglu else N
    g.lda, g.ldb = lda, ldb
    g.ldo = n_out if ldo is None else ldo
    g.ldr = n_out if ldr is None else ldr
    g.M, g.N, g.K = M, N, K
    if conv is not None:
        g.a_mode = 1
        g.img_n, g.img_h, g.img_w, g.img_c, g.ksize = conv
    else:
        g.a_mode = 0
    g.rows_per_vec = rows_per_vec
    g.out_kind = 0 if out.dtype == torch.float32 else 1
    g.act = ACT[act]
    g.act_param = act_param
    g.alpha = alpha
    g.geglu = int(geglu)
    g.force_bn = force_bn
    g.bias_per_row = 1 if bias_per_row else 0
    g.groups = groups
    if splitk_ws is not None:
        g.splitk_ws = splitk_ws.data_ptr()
        g.splitk_ws_bytes = splitk_ws.numel() * splitk_ws.element_size()
    g.split_k = split_k
    g.cta_pair = cta_pair
    g.gn_partials = _ptr(gn_partials)
    g.gn_rows_per_img = gn_rows_per_img
    check(lib.dbir_gemm(C.byref(g), C.c_void_p(stream_ptr())), "dbir_gemm")
    if _record is not None:
        keep = (a, b, out, bias, rowvec, residual, splitk_ws, gn_partials)     # keep buffers alive
        _record.append(("conv" if conv is not None else "gemm", (M, N, K), 2.0 * M * N * K,
                        lambda g=g, keep=keep: check(lib.dbir_gemm(C.byref(g), C.c_void_p(stream_ptr())), "dbir_gemm")))
    count_launch()


def _sp():
    return C.c_void_p(stream_ptr())


def _fp(t):
    return C.c_void_p(None if t is None else t.data_ptr())


def attention_ws_bytes(batch, heads, sq, skv) -> int:
    """Bytes of (zero-initialised, per-stream) workspace that let dbir_attention balance this
    shape over all SMs; 0 when whole tiles per CTA are used anyway."""
    lib = load()
    lib.dbir_attention_ws_bytes.restype = C.c_int64
    return int(lib.dbir_attention_ws_bytes(batch, heads, sq, skv))


def attention(q, k, v, out, *, batch, heads, sq, skv, ldq, ldk, ldv, ldo, ws=None):
    """Flash attention, head_dim 64; q/k/v/out are op16 tensors (possibly column slices).
    ws: optional zero-initialised uint8/float32 scratch of attention_ws_bytes() bytes."""
    ws_bytes = ws.numel() * ws.element_size() if ws is not None else 0

    def call():
        check(load().dbir_attention(_fp(q), _fp(k), _fp(v), _fp(out), batch, heads, sq, skv,
                                    C.c_int64(ldq), C.c_int64(ldk), C.c_int64(ldv), C.c_int64(ldo),
                                    _fp(ws), C.c_int64(ws_bytes), _sp()), "dbir_attention")
    call()
    if _record is not None:
        _record.append(("attention", (batch, heads, sq, skv), 4.0 * batch * heads * sq * skv * 64, call))
    count_launch()


def gn_workspace_floats(n, hw, c) -> int:
    lib = load()
    lib.dbir_gn_workspace_floats.restype = C.c_int64
    return int(lib.dbir_gn_workspace_floats(n, hw, c))


def gemm_gn_slots(conv_h=0, conv_w=0, rows_per_img=0) -> int:
    return int(load().dbir_gemm_gn_slots(conv_h, conv_w, rows_per_img))


def gn_finalize(p1, slots1, c1, p2, slots2, c2, n, hw, eps, stats):
    check(load().dbir_gn_finalize(_fp(p1), slots1, c1, _fp(p2), slots2, c2, n, hw, C.c_float(eps), _fp(stats),
                                  _sp()), "dbir_gn_finalize")
    count_launch()


def gn_stats(src1, src2, c1, c2, n, hw, eps, stats, workspace):
    check(load().dbir_gn_stats(_fp(src1), _fp(src2), c1, c2, n, hw, C.c_float(eps), _fp(stats),
                               _fp(workspace), _sp()), "dbir_gn_stats")
    count_launch()


def gn_moments_workspace_floats(n, hw, c) -> int:
    lib = load()
    lib.dbir_gn_moments_workspace_floats.restype = C.c_int64
    return int(lib.dbir_gn_moments_workspace_floats(n, hw, c))


def gn_moments(c, n, hw, moments, *, partials=None, slots=0, x=None, workspace=None, entry=None, entry0=0):
    """fp64 (mean, biased var) per (batch entry, group) of GEMM partial sums or a fp32 NHWC tensor x."""
    check(load().dbir_gn_moments(_fp(partials), slots, _fp(x), c, n, hw, _fp(workspace), _fp(entry), entry0,
                                 _fp(moments), _sp()), "dbir_gn_moments")
    count_launch(1 if x is None else 2)


def gn_merge(moments, pixels, image, entries, images, stats, *, reverse=False, eps=1e-6):
    """Tiled-VAE GroupNorm statistics: pixel-weighted mean of the entries' moments per (image, group)."""
    check(load().dbir_gn_merge(_fp(moments), _fp(pixels), _fp(image), entries, images, 1 if reverse else 0,
                               C.c_float(eps), _fp(stats), _sp()), "dbir_gn_merge")
    count_launch()


def gn_apply(src1, src2, c1, c2, n, h, w, stats, gamma, beta, out, *, norm=True, silu=True,
             upsample=1, out_raw=None, imgs_per_group=0):
    check(load().dbir_gn_apply(_fp(src1), _fp(src2), c1, c2, n, h, w, _fp(stats), _fp(gamma),
                               _fp(beta), 1 if norm else 0, 1 if silu else 0, upsample, _fp(out),
                               _fp(out_raw), imgs_per_group, _sp()), "dbir_gn_apply")
    count_launch()


def layernorm(x, ldx, rows, c, gamma, beta, out, ldo, eps=1e-5, rows_per_group=0):
    check(load().dbir_layernorm(_fp(x), C.c_int64(ldx), rows, c, _fp(gamma), _fp(beta),
                                C.c_float(eps), _fp(out), C.c_int64(ldo),
                                0 if out.dtype == torch.float32 else 1, rows_per_group, _sp()), "dbir_layernorm")
    count_launch()


def window_attention(qkv, ldq, batch, h, w, heads, head_dim, shift, bias_table, mask_value, out, ldo, window=8):
    check(load().dbir_window_attention(_fp(qkv), C.c_int64(ldq), batch, h, w, heads, head_dim, window, shift,
                                       _fp(bias_table), C.c_float(mask_value), _fp(out), C.c_int64(ldo), _sp()),
          "dbir_window_attention")
    count_launch()


def swin_patch_merge(x, ldx, n, h, w, c, gamma, beta, out, ldo, eps=1e-5):
    """Swin PatchMerging gather + LayerNorm over 4c: fp32 x [n*h*w, ldx] -> op16 out [n*h/2*w/2, ldo]."""
    check(load().dbir_swin_patch_merge(_fp(x), C.c_int64(ldx), n, h, w, c, _fp(gamma), _fp(beta), C.c_float(eps),
                                       _fp(out), C.c_int64(ldo), _sp()), "dbir_swin_patch_merge")
    count_launch()


def token_mean(x, ldx, n, tokens, c, out, ldo):
    """fp32 x [n*tokens, ldx] -> op16 out [n*(tokens+1), ldo]: per image [mean of its tokens | the tokens]."""
    check(load().dbir_token_mean(_fp(x), C.c_int64(ldx), n, tokens, c, _fp(out), C.c_int64(ldo), _sp()),
          "dbir_token_mean")
    count_launch()


def label_reweight(cls, ld_cls, batch, label_embed, classes, per_class, scale, out, ldo):
    """RAM++ description reweighting: out[b*classes + k] = sum_j softmax_j(scale * cls_b/|cls_b| . e_kj) e_kj."""
    check(load().dbir_label_reweight(_fp(cls), C.c_int64(ld_cls), batch, _fp(label_embed), classes, per_class,
                                     label_embed.shape[-1], C.c_float(scale), _fp(out), C.c_int64(ldo), _sp()),
          "dbir_label_reweight")
    count_launch()


def conv3x3_small_cin(in1, in2, c1, c2, n, h, w, weight_kc, bias, cout, out, in_scale=1.0,
                      in_shift=0.0):
    check(load().dbir_conv3x3_small_cin(_fp(in1), _fp(in2), c1, c2, n, h, w, _fp(weight_kc),
                                        _fp(bias), cout, C.c_float(in_scale), C.c_float(in_shift),
                                        _fp(out), _sp()), "dbir_conv3x3_small_cin")
    count_launch()


def conv3x3_small_cout(x, n, h, w, cin, weight, bias, cout, out, *, nchw=True, post_scale=1.0,
                       post_shift=None):
    check(load().dbir_conv3x3_small_cout(_fp(x), n, h, w, cin, _fp(weight), _fp(bias), cout,
                                         C.c_float(post_scale), _fp(post_shift), _fp(out),
                                         1 if nchw else 0, _sp()), "dbir_conv3x3_small_cout")
    count_launch()


def im2col_s2(x, n, h, w, c, pad_lo, out):
    check(load().dbir_im2col_s2(_fp(x), n, h, w, c, pad_lo, _fp(out), _sp()), "dbir_im2col_s2")
    count_launch()


def linear_f32(x, ldx, m, k, weight, bias, n, y, ldy, silu_in=False, silu_out=False):
    check(load().dbir_linear_f32(_fp(x), C.c_int64(ldx), m, k, _fp(weight), _fp(bias), n,
                                 1 if silu_in else 0, 1 if silu_out else 0, _fp(y),
                                 C.c_int64(ldy), _sp()), "dbir_linear_f32")
    count_launch()


def axpby_cast(x, alpha, z, rows, c, y=None, y16=None, ld16=0):
    check(load().dbir_axpby_cast(_fp(x), C.c_float(alpha), _fp(z), C.c_int64(rows), c, _fp(y), _fp(y16),
                                 C.c_int64(ld16), _sp()), "dbir_axpby_cast")
    count_launch()


def timestep_embedding(t, m, dim, out):
    check(load().dbir_timestep_embedding(_fp(t), m, dim, _fp(out), _sp()), "dbir_timestep_embedding")
    count_launch()


def softmax_rows(s, lds, rows, cols, scale, out, ldo):
    check(load().dbir_softmax_rows(_fp(s), C.c_int64(lds), rows, cols, C.c_float(scale), _fp(out),
                                   C.c_int64(ldo), _sp()), "dbir_softmax_rows")
    count_launch()


def upsample2x_op16(x, n, h, w, c, out):
    check(load().dbir_upsample2x_op16(_fp(x), n, h, w, c, _fp(out), _sp()), "dbir_upsample2x_op16")
    count_launch()


def swin_stem(x, n, h, w, r, mean3, rng, cpad, out):
    arr = (C.c_float * 3)(*mean3)
    check(load().dbir_swin_stem(_fp(x), n, h, w, r, arr, C.c_float(rng), cpad, _fp(out), _sp()),
          "dbir_swin_stem")
    count_launch()


def nchw_to_nhwc(x, n, c, hw, out):
    check(load().dbir_nchw_to_nhwc(_fp(x), n, c, hw, _fp(out), _sp()), "dbir_nchw_to_nhwc")
    count_launch()


def nhwc_to_nchw(x, n, c, hw, out):
    check(load().dbir_nhwc_to_nchw(_fp(x), n, c, hw, _fp(out), _sp()), "dbir_nhwc_to_nchw")
    count_launch()


def sampler_step(eps_c, eps_u, cfg, x, noise, coef, mode, numel, x_out):
    check(load().dbir_sampler_step(_fp(eps_c), _fp(eps_u), C.c_float(cfg), _fp(x), _fp(noise),
                                   _fp(coef), mode, C.c_int64(numel), _fp(x_out), _sp()),
          "dbir_sampler_step")
    count_launch()


def tile_gather(full, b, c, h, w, coords, ntiles, tile, tiles):
    check(load().dbir_tile_gather(_fp(full), b, c, h, w, _fp(coords), ntiles, tile, _fp(tiles),
                                  _sp()), "dbir_tile_gather")
    count_launch()


def tile_blend(tiles, b, c, h, w, coords, ntiles, tile, weights, out):
    check(load().dbir_tile_blend(_fp(tiles), b, c, h, w, _fp(coords), ntiles, tile, _fp(weights),
                                 _fp(out), _sp()), "dbir_tile_blend")
    count_launch()


def wavelet_fix(sample, style, out_u8=None, out_f32=None):
    """Fused colour fix (+ uint8 quantisation): sample NCHW view in [-1, 1], style NCHW view in [0, 1],
    both fp32 with unit column stride; exactly one of out_u8 (NHWC uint8) / out_f32 (NCHW fp32)."""
    b, c, h, w = sample.shape
    assert c == 3 and tuple(style.shape) == (b, c, h, w) and sample.stride(3) == 1 and style.stride(3) == 1
    i64 = C.c_int64
    check(load().dbir_wavelet_fix(_fp(sample), i64(sample.stride(0)), i64(sample.stride(1)), i64(sample.stride(2)),
                                  _fp(style), i64(style.stride(0)), i64(style.stride(1)), i64(style.stride(2)),
                                  b, h, w, _fp(out_u8), _fp(out_f32), _sp()), "dbir_wavelet_fix")
    count_launch()


# ---- face detector / face parser (include/diffbir_b200.h, "face detector / face parser") ----
def face_input(img_u8, n, h, w, out, *, scale=1.0, shift=(0.0, 0.0, 0.0), div=1.0, reverse=False):
    check(load().dbir_face_input(_fp(img_u8), n, h, w, C.c_float(scale), C.c_float(shift[0]), C.c_float(shift[1]),
                                 C.c_float(shift[2]), C.c_float(div), 1 if reverse else 0, _fp(out), _sp()),
          "dbir_face_input")
    count_launch()


def patch_gather_shape(h, w, ksize, stride, up2=False):
    """(ho, wo) of dbir_patch_gather's output grid."""
    hs, ws, pad = (2 * h, 2 * w, ksize // 2) if up2 else (h, w, ksize // 2)
    return (hs + 2 * pad - ksize) // stride + 1, (ws + 2 * pad - ksize) // stride + 1


def patch_gather(x, ldx, n, h, w, c, ksize, stride, kpad, out, *, reflect=False, up2=False):
    check(load().dbir_patch_gather(_fp(x), C.c_int64(ldx), n, h, w, c, ksize, stride, 1 if reflect else 0,
                                   1 if up2 else 0, kpad, _fp(out), _sp()), "dbir_patch_gather")
    count_launch()


def maxpool3s2(x, n, h, w, c, out):
    check(load().dbir_maxpool3s2(_fp(x), n, h, w, c, _fp(out), _sp()), "dbir_maxpool3s2")
    count_launch()


def fpn_add_up(a, b, n, h, w, hb, wb, c, out):
    check(load().dbir_fpn_add_up(_fp(a), _fp(b), n, h, w, hb, wb, c, _fp(out), _sp()), "dbir_fpn_add_up")
    count_launch()


def relu_cast(x, numel, y16, y=None):
    check(load().dbir_relu_cast(_fp(x), C.c_int64(numel), _fp(y), _fp(y16), _sp()), "dbir_relu_cast")
    count_launch()


def retinaface_decode(head, h, w, out):
    check(load().dbir_retinaface_decode(_fp(head), h, w, _fp(out), _sp()), "dbir_retinaface_decode")
    count_launch()


def parse_mask(logits, ld, rows, classes, out):
    check(load().dbir_parse_mask(_fp(logits), C.c_int64(ld), C.c_int64(rows), classes, _fp(out), _sp()),
          "dbir_parse_mask")
    count_launch()


# ---- LLaVA captioner language model (include/diffbir_b200.h, "LLaVA captioner language model") ----
def rmsnorm(x, ldx, rows, c, w, out, ldo, eps=1e-5):
    check(load().dbir_rmsnorm(_fp(x), C.c_int64(ldx), rows, c, _fp(w), C.c_float(eps), _fp(out), C.c_int64(ldo), _sp()),
          "dbir_rmsnorm")
    count_launch()


def rope_kv(qkv, ldqkv, rows, heads, p0, q, ldq, k_cache, v_cache, theta=10000.0):
    check(load().dbir_rope_kv(_fp(qkv), C.c_int64(ldqkv), rows, heads, _fp(p0), C.c_float(theta), _fp(q), C.c_int64(ldq),
                              _fp(k_cache), _fp(v_cache), _sp()), "dbir_rope_kv")
    count_launch()


def attention_causal(q, ldq, k_cache, v_cache, heads, sq, out, ldo):
    check(load().dbir_attention_causal(_fp(q), C.c_int64(ldq), _fp(k_cache), _fp(v_cache), heads, sq, _fp(out),
                                       C.c_int64(ldo), _sp()), "dbir_attention_causal")
    count_launch()


def attention_decode_ws_bytes(heads, capacity) -> int:
    lib = load()
    lib.dbir_attention_decode_ws_bytes.restype = C.c_int64
    return int(lib.dbir_attention_decode_ws_bytes(heads, capacity))


def attention_decode(q, k_cache, v_cache, heads, capacity, length, ws, out):
    """length: device int32 [1] holding the number of cache rows to attend to."""
    check(load().dbir_attention_decode(_fp(q), _fp(k_cache), _fp(v_cache), heads, capacity, _fp(length), _fp(ws),
                                       C.c_int64(ws.numel() * ws.element_size()), _fp(out), _sp()),
          "dbir_attention_decode")
    count_launch(2)


GEMV_EPILOGUE = {"none": 0, "residual": 1, "swiglu": 2}


def gemv(w, x, y, *, N, K, ldw=0, epilogue="none", pack=0, residual=None):
    """y = W x for one row (op16 W [N, ldw], op16 x [K]); y fp32 or op16. epilogue: none / residual / swiglu."""
    check(load().dbir_gemv(_fp(w), C.c_int64(ldw or K), _fp(x), N, K, GEMV_EPILOGUE[epilogue], pack, _fp(residual),
                           _fp(y), 0 if y.dtype == torch.float32 else 1, _sp()), "dbir_gemv")
    count_launch()


def argmax(logits, n, token, advance=None):
    """First maximum of fp32 logits [n] -> device int32 token; each element of `advance` (device int32) += 1."""
    n_adv = 0 if advance is None else advance.numel()
    check(load().dbir_argmax(_fp(logits), n, _fp(token), _fp(advance), n_adv, _sp()), "dbir_argmax")
    count_launch()


def embed_gather(table, vocab, ids, n, dim, out, ldo):
    check(load().dbir_embed_gather(_fp(table), vocab, _fp(ids), n, dim, _fp(out), C.c_int64(ldo), _sp()),
          "dbir_embed_gather")
    count_launch()
