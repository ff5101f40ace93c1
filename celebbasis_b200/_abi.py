"""ctypes signatures of every non-GEMM entry point of include/celebbasis_b200.h."""
import ctypes as C

_p, _i, _l, _f = C.c_void_p, C.c_int32, C.c_longlong, C.c_float

SIGS = {
    "cb_groupnorm_cluster_plan": [_i, _i, _i, _i, _i, _p],
    "cb_groupnorm_fwd": [_p, _i, _p, _i, _p, _p, _i, _i, _i, _i, _f, _i, _p, _p, _p, _p],
    "cb_groupnorm_bwd": [_p, _i, _p, _i, _p, _p, _p, _p, _p, _i, _p, _i, _i, _i, _i, _i, _i, _p, _p],
    "cb_layernorm_fwd": [_p, _i, _p, _i, _p, _p, _i, _i, _f, _p, _p, _p],
    "cb_layernorm_bwd": [_p, _i, _p, _i, _p, _p, _p, _p, _i, _p, _i, _i, _i, _p],
    "cb_axpby2d": [_p, _i, _l, _f, _p, _i, _l, _f, _p, _i, _l, _l, _i, _p],
    "cb_act_fwd": [_p, _i, _p, _i, _l, _i, _p],
    "cb_act_bwd": [_p, _i, _p, _i, _p, _i, _l, _i, _p],
    "cb_geglu_fwd": [_p, _p, _i, _l, _i, _i, _p],
    "cb_geglu_bwd": [_p, _p, _p, _i, _i, _l, _i, _i, _p],
    "cb_softmax_fwd": [_p, _p, _i, _l, _i, _i, _i, _p],
    "cb_softmax_bwd": [_p, _p, _p, _i, _i, _l, _i, _i, _p],
    "cb_upsample2x_fwd": [_p, _p, _i, _i, _i, _i, _i, _p],
    "cb_upsample2x_bwd": [_p, _i, _p, _i, _i, _i, _i, _i, _i, _p],
    "cb_zero_insert2x": [_p, _p, _i, _i, _i, _i, _i, _p],
    "cb_nchw_to_nhwc": [_p, _p, _i, _i, _i, _i, _i, _p],
    "cb_nhwc_to_nchw": [_p, _i, _p, _i, _i, _i, _i, _p],
    "cb_mse_fwd_bwd": [_p, _p, _p, _p, _i, _i, _f, _p],
    "cb_timestep_embedding": [_p, _p, _i, _i, _i, _f, _p],
    "cb_embedding_gather": [_p, _p, _p, _i, _i, _i, _p],
    "cb_celeb_mlp_fwd": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _f, _p],
    "cb_celeb_basis_fwd": [_p, _p, _p, _i, _i, _i, _i, _p],
    "cb_celeb_basis_bwd": [_p, _p, _p, _i, _i, _i, _i, _p],
    "cb_celeb_mlp_bwd": [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _f, _f, _p],
    "cb_embed_inject_fwd": [_p, _p, _p, _p, _p, _i, _i, _i, _p],
    "cb_embed_inject_bwd": [_p, _p, _p, _i, _i, _i, _i, _p],
    "cb_adamw_step": [_p, _p, _p, _p, _l, _f, _f, _f, _f, _f, _i, _p, _p],
    "cb_posterior_sample": [_p, _p, _p, _i, _i, _i, _f, _p],
    "cb_loss_mean": [_p, _p, _i, _p],
    "cb_diffusion_loss_fwd_bwd": [_p, _p, _p, _p, _p, _f, _f, _p, _p, _p, _p, _i, _i, _f, _p],
    "cb_ti_coarse_reg": [_p, _p, _p, _p, _i, _i, _i, _f, _p],
    "cb_ddim_step": [_p, _p, _p, _p, _p, _p, _l, _f, _f, _f, _f, _f, _p],
    "cb_attention_fwd": [_p, _l, _p, _l, _p, _l, _p, _l, _p, _p, _l, _i, _i, _i, _i, _i, _i, _f, _i, _p],
    "cb_attention_bwd": [_p, _l, _p, _l, _p, _l, _p, _l, _p, _l, _p, _p, _p, _l, _p, _l, _p, _l, _i, _i, _i, _i, _i, _i, _f,
                         _i, _p],
    "cb_attention_bwd_dq": [_p, _l, _p, _l, _p, _l, _p, _l, _p, _l, _p, _p, _p, _l, _p, _l, _i, _i, _i, _i, _i, _i, _f, _i, _p],
    "cb_q_sample": [_p, _p, _p, _p, _p, _p, _i, _i, _p],
    "cb_q_sample_masked": [_p, _p, _p, _p, _p, _p, _l, _l, _p, _p, _i, _i, _i, _p],
    "cb_p_sample": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _f, _i, _p, _p, _i, _i, _p],
    "cb_channel_affine_act": [_p, _i, _p, _i, _p, _p, _p, _l, _i, _p],
    "cb_face_warp_resize": [_p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p],
    "cb_l2norm_rows": [_p, _p, _i, _i, _p],
    "cb_ema_rows": [_p, _p, _i, _p, _i, _i, _i, _f, _p],
    "cb_ema_rows_sel": [_p, _p, _p, _p, _p, _i, _i, _i, _f, _p],
    "cb_face_augment": [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    "cb_paste_resized": [_p, _i, _i, _p, _p, _i, _i, _i, _p],
    "cb_pack_conv_weight": [_p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p],
    "cb_convert_f32": [_p, _p, _i, _l, _f, _p],
}


def declare(lib):
    for name, argtypes in SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
