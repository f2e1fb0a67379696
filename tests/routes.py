"""Route keys: which kernel instantiation each es3_* call selects, and which test files hold every instantiation to its bounds.

KEYS maps every kernel entry point of include/es3.h to a function of the call's arguments.  A key is the entry point's name
followed by what its arguments select (tile, template width, activation, optional operands present ...); an entry point whose
arguments select nothing finer has the name-only key (name,).  Keys of different entry points therefore never collide.

COVERED names, for every entry point, the test files whose tables run it.  A file that defines covered_keys() covers exactly the
keys that function returns; any other file covers the name-only key of the entry points it is listed for.

assert_closed(calls, who) is the route closure: every call a real model path makes (tests/es3_recorder.py records them) must have a
key function, and its key must be covered by a file listed for its entry point.  So the fp64 tables test what the models run.
"""
import importlib
from collections import defaultdict

from ref_vit import bn_tile

HOST_ONLY = {"es3_init", "es3_version", "es3_last_error"}       # and the *_ws_floats size queries: no kernel behind them
_ACT = {0: None, 1: "relu", 2: "hswish", 3: "gelu", 6: "sigmoid"}
_BN_MODE = {0: "none", 1: "eval", 2: "batch"}


def is_kernel(name):
    return name not in HOST_ONLY and not name.endswith("_ws_floats")


def _act(code):
    return _ACT.get(code, code)


def _nz(x):
    return x not in (None, 0)


# ----------------------------------------------------------------------------------------------------------- key helpers
def dw_tc_key(ks, C, act):
    return ("es3_dwconv_tc_bf16", ks, 64 if ks == 3 and C % 64 == 0 else 32, act)


def ln_key(C):
    nv = C // 8
    return ("es3_layernorm_bf16", 8 if nv <= 8 else (16 if nv <= 16 else 32))


def wg_pick(c):
    return 1 if c <= 16 else (2 if c <= 32 else 4)


def key_wgrad_pw(N, K, shifted):
    return ("es3_wgrad_pw", wg_pick(N), wg_pick(K), "shift" if shifted else "plain")


def key_wgrad_tc(K):
    return ("es3_wgrad_tc", 128 if K >= 128 else 64)


def key_dw_bwd_data(ks, stride):
    return ("es3_dwconv_bwd_data", "s2k3" if (ks, stride) == (3, 2) else "generic", ks, stride)


def attn_key(name, H, W, win):
    """es3_attention_bf16 and the two kernels it dispatches to: (name, kernel, key tile (wgmma) or MT (mma.sync), windowed)."""
    L = win * win if win else H * W
    if name == "es3_attention_tc_bf16" or (name == "es3_attention_bf16" and L >= 128):
        return (name, "tc", bn_tile(L), win > 0)
    return (name, "mma", 2 if L >= 128 else 1, win > 0)


def causal_attn_key(L):
    return ("es3_attention_causal_bf16", 2 if L >= 128 else 1)


# The wgmma GEMM family (gemm_tc.cu) selects gemm_tc_kernel<BN, STAGES, ACT> by the rules restated here.  In its keys activations
# go by name, residuals and outputs by dtype ("bf16" / "f32", None when absent), RoPE as None / "window" / "global".
def pick_bn(N, bn_hint, K=1 << 30, act=None):
    """gemm_tc.cu pick_bn: the tile width for N output columns, a tile-width hint, K and the activation."""
    if bn_hint in (32, 64, 128):
        return bn_hint
    if bn_hint == 256:
        return 128
    if K < 512 and N >= 64:
        if act == "gelu":
            return 64
        return 128 if N >= 384 else 64
    if N % 128 == 0 or N > 1024:
        return 128
    if N % 64 == 0:
        return 64
    return 128 if N >= 128 else 32


def gemm_bn(N, K, act, rope, bn_hint):
    """es3_gemm_bf16_ex: pick_bn, except that the RoPE epilogue takes 128-wide tiles when N >= 128 and no hint is given."""
    return 128 if rope is not None and bn_hint == 0 and N >= 128 else pick_bn(N, bn_hint, K, act)


def gemm_stages(bn, num_kb):
    """gemm_tc.cu dispatch: the operand ring's depth at tile width bn for num_kb 64-wide k-blocks."""
    if bn == 128:
        return 2 if num_kb <= 2 else 4
    return 2 if bn == 64 else 4


def conv_tile_w(W):
    """es3_conv3x3_bf16: the implicit GEMM's tile width in pixels for an image W pixels wide."""
    return 32 if W % 32 == 0 else (16 if W % 16 == 0 else 8)


def conv3x3_num_kb(C):
    """es3_conv3x3_bf16: nine taps of ceil(C / 64) k-blocks each."""
    return 9 * -(-C // 64)


def gemm_key(name, N, K, act, scale, bias, res, after, out, rope, bn_hint):
    """es3_gemm_bf16_ex / es3_gemm_bf16: (name, BN, STAGES, act, scale, bias, residual, act after the residual (only when both are
    present), out, RoPE, ragged last 32-column chunk)."""
    bn = gemm_bn(N, K, act, rope, bn_hint)
    return (name, bn, gemm_stages(bn, -(-K // 64)), act, bool(scale), bool(bias), res, bool(after and res and act), out, rope,
            N % 32 != 0)


def conv3x3_key(N, W, act, scale, bias, res, out, bn_hint):
    return ("es3_conv3x3_bf16", pick_bn(N, bn_hint), conv_tile_w(W), act, bool(scale), bool(bias), res, out)


def convt2x2_key(Cin, Cout, act, res, after, out):
    bn = pick_bn(4 * Cout, 0)
    return ("es3_convt2x2_bf16", bn, gemm_stages(bn, -(-Cin // 64)), act, res, bool(after and res and act), out)


def fp8_attn_key(H, W, win):
    """es3_attention_fp8: the key tile is 96 when L is a multiple of 96 but not of 128 (attention_fp8.cu), else 128."""
    L = win * win if win else H * W
    return ("es3_attention_fp8", 96 if L % 96 == 0 and L % 128 != 0 else 128, win > 0)


def grad_norm_key(n):
    """es3_grad_norm: (name, ragged n % 4, grid capped: more than 4096 blocks of 16384 elements, so threads loop)."""
    return ("es3_grad_norm", n % 4 != 0, -(-n // 16384) > 4096)


def adamw_key(n, n_decay, max_norm, dynamic):
    """es3_adamw_flat: (name, clipping on, dynamic loss scale, ragged n % 4, decay split 0 < n_decay < n)."""
    return ("es3_adamw_flat", max_norm > 0, bool(dynamic), n % 4 != 0, 0 < n_decay < n)


def _res(ptr, f32):
    return ("f32" if f32 else "bf16") if _nz(ptr) else None


def _dt(f32):
    return "f32" if f32 else "bf16"


def _rope(ptr, win):
    return ("window" if win else "global") if _nz(ptr) else None


# ----------------------------------------------------------------------------------------------------------- KEYS
_DETAILED = {
    # image students' forward kernels
    "es3_mbconv_bf16": lambda a: ("es3_mbconv_bf16", a[13], a[14], a[15], a[16]),
    "es3_dwproj_tc_bf16": lambda a: ("es3_dwproj_tc_bf16", a[11], a[12]),
    "es3_dwconv_tc_bf16": lambda a: dw_tc_key(a[10], a[9], _act(a[11])),
    "es3_dwconv_tiled_bf16": lambda a: ("es3_dwconv_tiled_bf16", a[10], a[11], _act(a[12])),
    "es3_dwconv_bf16": lambda a: ("es3_dwconv_bf16", a[10], a[11], _act(a[12])),
    "es3_stem_conv3x3_s2": lambda a: ("es3_stem_conv3x3_s2", a[7], _act(a[8])),
    "es3_dsconv_res_bf16": lambda a: ("es3_dsconv_res_bf16", a[9], _act(a[10])),
    "es3_litemla_attn_generic": lambda a: ("es3_litemla_attn_generic", a[8]),
    "es3_conv3x3_s2_narrow_bf16": lambda a: ("es3_conv3x3_s2_narrow_bf16", a[8], a[9], _act(a[10])),
    "es3_win_attn_bias_bf16": lambda a: ("es3_win_attn_bias_bf16", a[9]),
    "es3_layernorm_bf16": lambda a: ln_key(a[6]),
    # image students' backward kernels
    "es3_wgrad_pw": lambda a: key_wgrad_pw(a[5], a[6], a[7] > 0),
    "es3_wgrad_tc": lambda a: key_wgrad_tc(a[6]),
    "es3_dwconv_bwd_data": lambda a: key_dw_bwd_data(a[7], a[8]),
    "es3_dwconv_wgrad": lambda a: ("es3_dwconv_wgrad", a[7], a[8]),
    "es3_dwconv_wgrad_win": lambda a: ("es3_dwconv_wgrad_win", a[7], a[8]),
    "es3_bn_act_bwd_reduce": lambda a: ("es3_bn_act_bwd_reduce", _act(a[4]), _BN_MODE[a[5]], a[2] != 0),
    "es3_bn_act_bwd_apply": lambda a: ("es3_bn_act_bwd_apply", _act(a[4]), a[2] != 0),
    "es3_affine_act": lambda a: ("es3_affine_act", _act(a[3]), a[1] != 0, a[4] != 0),
    "es3_stem_wgrad": lambda a: ("es3_stem_wgrad", a[5]),
    "es3_litemla_attn_bwd_generic": lambda a: ("es3_litemla_attn_bwd_generic", a[12]),
    "es3_layernorm_bwd": lambda a: ("es3_layernorm_bwd", a[3] != 0),
    "es3_win_attn_bias_bwd": lambda a: ("es3_win_attn_bias_bwd", a[11]),
    # text encoders
    "es3_attention_causal_bf16": lambda a: causal_attn_key(a[3]),
    "es3_text_attn_bwd": lambda a: ("es3_text_attn_bwd", bool(a[8])),
    "es3_layernorm_f32": lambda a: ("es3_layernorm_f32", a[11] // 128),
    "es3_layernorm_bwd_f32": lambda a: ("es3_layernorm_bwd_f32", _nz(a[3]), _nz(a[6]), a[7] > 37888),
    "es3_text_pos_grad": lambda a: ("es3_text_pos_grad", a[2] == a[3]),
    "es3_text_kd_loss_fwd": lambda a: ("es3_text_kd_loss_fwd", _nz(a[2])),
    "es3_text_kd_loss_bwd": lambda a: ("es3_text_kd_loss_bwd", _nz(a[2]), _nz(a[9]), _nz(a[10])),
    "es3_text_consistency_bwd": lambda a: ("es3_text_consistency_bwd", _nz(a[6]), _nz(a[7])),
    # SAM heads
    "es3_point_embed": lambda a: ("es3_point_embed", _nz(a[8])),
    "es3_add_rows": lambda a: ("es3_add_rows", _nz(a[1]), _nz(a[5]), _nz(a[6])),
    "es3_nchw_f32_to_tokens": lambda a: ("es3_nchw_f32_to_tokens", _nz(a[1]), _nz(a[2])),
    "es3_attn_few_queries": lambda a: ("es3_attn_few_queries", a[10], bool(a[5])),
    "es3_attn_few_keys": lambda a: ("es3_attn_few_keys", a[11] > 16),
    "es3_attn_few_keys_f32": lambda a: ("es3_attn_few_keys_f32", a[11] > 16),
    "es3_ln_rows_gelu": lambda a: ("es3_ln_rows_gelu", a[6]),
    "es3_ln_rows_gelu_f32": lambda a: ("es3_ln_rows_gelu_f32", a[6]),
    "es3_hyper_masks": lambda a: ("es3_hyper_masks", _nz(a[2]), a[9], a[10]),
    "es3_bilinear_nchw_f32": lambda a: ("es3_bilinear_nchw_f32", _nz(a[1]), _nz(a[2])),
    "es3_mask_downscale_tokens": lambda a: ("es3_mask_downscale_tokens", _nz(a[11]), _nz(a[13]), _nz(a[14])),
    # SAM3 ViT trunk
    "es3_attention_bf16": lambda a: attn_key("es3_attention_bf16", a[3], a[4], a[7]),
    "es3_attention_tc_bf16": lambda a: attn_key("es3_attention_tc_bf16", a[3], a[4], a[7]),
    "es3_attention_mma_bf16": lambda a: attn_key("es3_attention_mma_bf16", a[3], a[4], a[7]),
    "es3_sgemm_f32": lambda a: ("es3_sgemm_f32", a[11], bool(a[14]), _nz(a[9]), _nz(a[10]), _nz(a[12])),
    "es3_rope_f32": lambda a: ("es3_rope_f32", a[7] > 0),
    "es3_attention_f32": lambda a: ("es3_attention_f32", a[9], _nz(a[2]), _nz(a[3]), a[14] > 0),
    "es3_im2col_f32": lambda a: ("es3_im2col_f32", bool(a[9]), a[6], a[7]),
    # the strict mode's student kernels
    "es3_dwconv_f32": lambda a: ("es3_dwconv_f32", a[11], a[12], _act(a[13]), _nz(a[3]), _nz(a[4])),
    "es3_litemla_attn_f32": lambda a: ("es3_litemla_attn_f32", a[8], a[6] > 2048),          # HW > 2048: more than one chunk
    "es3_bias_act_res_f32": lambda a: ("es3_bias_act_res_f32", _act(a[6]), _nz(a[1]), _nz(a[2]), bool(a[7])),
    "es3_bilinear_nhwc_f32_to_nchw": lambda a: ("es3_bilinear_nhwc_f32_to_nchw", "same" if (a[3], a[4]) == (a[6], a[7]) else "resize"),
    # GEMMs and convolutions on the wgmma GEMM, the narrow pointwise and CUDA-core GEMMs
    "es3_gemm_bf16_ex": lambda a: gemm_key("es3_gemm_bf16_ex", a[8], a[9], _act(a[12]), _nz(a[10]), _nz(a[11]), _res(a[13], a[15]),
                                           a[21], _dt(a[6]), _rope(a[16], a[20]), a[22]),
    "es3_gemm_bf16": lambda a: gemm_key("es3_gemm_bf16", a[8], a[9], _act(a[12]), _nz(a[10]), _nz(a[11]), _res(a[13], 0), False,
                                        _dt(a[6]), None, a[15]),
    "es3_conv3x3_bf16": lambda a: conv3x3_key(a[8], a[6], _act(a[11]), _nz(a[9]), _nz(a[10]), _res(a[12], 0), _dt(a[3]), a[13]),
    "es3_convt2x2_bf16": lambda a: convt2x2_key(a[7], a[8], _act(a[10]), _res(a[11], a[12]), a[13], _dt(a[3])),
    "es3_pw_small_bf16": lambda a: ("es3_pw_small_bf16", a[10], a[9], _nz(a[6])),
    "es3_gemm_simt": lambda a: ("es3_gemm_simt", _dt(a[2]), _dt(a[5]), _act(a[14]), _nz(a[12]), _nz(a[13]), _res(a[15], a[17]),
                                _dt(a[8])),
    # the SAM3 ViT teacher's FP8 route
    "es3_gemm_fp8": lambda a: ("es3_gemm_fp8", ("bf16", "f32", "e4m3")[a[8]], _act(a[14]), _nz(a[15]), _rope(a[17], a[21])),
    "es3_attention_fp8": lambda a: fp8_attn_key(a[4], a[5], a[8]),
    "es3_pack_weight_e4m3": lambda a: ("es3_pack_weight_e4m3", _dt(a[1])),
    "es3_layernorm_f32_e4m3": lambda a: ("es3_layernorm_f32_e4m3", a[7] // 128),
    # the stage-1 KD loss and optimiser
    "es3_kd_loss_fwd": lambda a: ("es3_kd_loss_fwd", _nz(a[10])),                                  # per_sample present
    "es3_kd_loss_bwd": lambda a: ("es3_kd_loss_bwd", _nz(a[4])),                                   # scale_dev present
    "es3_grad_norm": lambda a: grad_norm_key(a[1]),
    "es3_adamw_flat": lambda a: adamw_key(a[4], a[5], a[11], a[15]),
}

_FWD, _BWD, _TEXT, _SAM, _VIT = ("test_fwd_kernels_gpu.py", "test_train_bwd_gpu.py", "test_text_kernels_gpu.py",
                                 "test_sam_kernels_gpu.py", "test_vit_kernels_gpu.py")
_GEMM, _STRICT, _STAGE1 = "test_gemm_epilogue_gpu.py", "test_strict_kernels_gpu.py", "test_stage1_kernels_gpu.py"
_FILES = {
    _FWD: """mbconv_bf16 dwproj_tc_bf16 dwconv_tc_bf16 dwconv_tiled_bf16 dwconv_bf16 stem_conv3x3_s2 dsconv_res_bf16 litemla_attn_generic
             conv3x3_s2_narrow_bf16 win_attn_bias_bf16 layernorm_bf16 stem_fused_c16 litemla_aggreg_dwpw litemla_attn_tc channel_mean
             scale_channels round_taps_sum_bf16 bilinear_nhwc_to_nchw maxpool2x2_bf16 nhwc_to_nchw_f32 nchw_f32_to_nhwc""",
    _BWD: """wgrad_pw wgrad_tc dwconv_bwd_data dwconv_wgrad dwconv_wgrad_win bn_act_bwd_reduce bn_act_bwd_apply affine_act stem_wgrad
             litemla_attn_bwd_generic layernorm_bwd win_attn_bias_bwd bn_stats add_bf16 se_bwd_dgate se_bwd_apply bilinear_bwd
             litemla_attn_bwd colsum_f32 transpose_pad_bf16 accumulate_strided""",
    _TEXT: """attention_bf16 attention_causal_bf16 text_attn_bwd layernorm_f32 layernorm_bwd_f32 text_pos_resize text_pos_grad
              text_kd_loss_fwd text_kd_loss_bwd text_consistency_fwd text_consistency_bwd text_embed text_embed_grad repmixer_bf16
              repmixer_ls_bwd repmixer_ffn_bwd repmixer_tm_bwd cast_f32_to_bf16 cast_f32_to_f16""",
    _SAM: """dense_pe point_embed add_rows nchw_f32_to_tokens attn_few_queries attn_few_keys attn_few_keys_f32 ln_rows_gelu
             ln_rows_gelu_f32 hyper_masks bilinear_nchw_f32 mask_downscale_tokens""",
    _VIT: """attention_bf16 attention_tc_bf16 attention_mma_bf16 sgemm_f32 rope_f32 attention_f32 im2col_f32 im2col_patch
             tokens_f32_to_nchw ln_rows_f32""",
    _STRICT: "dwconv_f32 litemla_attn_f32 bias_act_res_f32 bilinear_nhwc_f32_to_nchw scale_channels_f32",
    _GEMM: "gemm_bf16 gemm_bf16_ex pw_small_bf16 gemm_simt conv3x3_bf16 convt2x2_bf16",
    "test_fp8_gpu.py": "gemm_fp8 quantize_bf16_e4m3 pack_weight_e4m3 layernorm_f32_e4m3",
    "test_fp8_attention_gpu.py": "attention_fp8",
    _STAGE1: "kd_loss_fwd kd_loss_bwd grad_norm adamw_flat",
    # files without covered_keys(): they hold the name-only key of the entry points listed for them
    "test_amg_gpu.py": "amg_mask_stats box_nms amg_rle",
    "test_preprocess_gpu.py": "prepare_images_u8",
    "test_decoder_gpu.py": "fill_small_components",
    "test_syncbn_gpu.py": "bn_stats_partial bn_stats_combine bn_act_bwd_partial bn_bwd_coef",
    "test_syncbn_repmixer_gpu.py": """repmixer_bn_fwd repmixer_bn_stats_partial repmixer_bn_finalize_sync repmixer_bn_tm_sums
                                      repmixer_bn_tm_apply repmixer_bn_tm_bwd repmixer_bn_ffn_sums repmixer_bn_ffn_apply
                                      repmixer_bn_ffn_bwd""",
}
COVERED = defaultdict(list)                 # entry point -> the test files whose tables run it
for _f, _names in _FILES.items():
    for _n in _names.split():
        COVERED["es3_" + _n].append(_f)
COVERED = dict(COVERED)
KEYS = {n: (lambda a, n=n: (n,)) for n in COVERED} | _DETAILED


def covered_keys(file):
    """The route keys the tables of test file `file` run."""
    mod = importlib.import_module(file[:-len(".py")])
    if hasattr(mod, "covered_keys"):
        return mod.covered_keys()
    return {(n,) for n, files in COVERED.items() if file in files}


def assert_closed(calls, who):
    """Every recorded (name, args) call has a key function and its key is covered by a file listed for its entry point.  Prints the
    reached keys per covering file; returns the set of reached keys."""
    calls = [(n, a) for n, a in calls if is_kernel(n)]
    unknown = sorted({n for n, _ in calls if n not in KEYS})
    assert not unknown, f"{who} reaches entry points with no route key: {unknown}"
    cover = {}
    by_file = defaultdict(set)
    missing = set()
    for n, a in calls:
        key = KEYS[n](a)
        files = COVERED[n]
        for f in files:
            if f not in cover:
                cover[f] = covered_keys(f)
        owners = [f for f in files if key in cover[f]]
        if not owners:
            missing.add(key)
        by_file[owners[0] if owners else files[0]].add(key)
    for f in sorted(by_file):
        print(f"\n{who}: {len(by_file[f])} route keys of {f} reached: {sorted(by_file[f], key=repr)}", end="")
    assert not missing, f"{who} reaches routes no table row runs: {sorted(missing, key=repr)}"
    return set().union(*by_file.values()) if by_file else set()
