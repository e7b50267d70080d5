"""ctypes binding of libb200trk.so (the C ABI declared in include/b200trk.h).

There is NO fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200trk.so")

c_float_p = C.POINTER(C.c_float)
c_int64_p = C.POINTER(C.c_int64)


class ConvDesc(C.Structure):
    """b200trk_conv_desc_t"""
    _fields_ = [("weight", C.c_void_p), ("bias", C.c_void_p), ("bn_gamma", C.c_void_p), ("bn_beta", C.c_void_p),
                ("bn_mean", C.c_void_p), ("bn_var", C.c_void_p),
                ("cout", C.c_int), ("cin", C.c_int), ("k", C.c_int), ("stride", C.c_int), ("pad", C.c_int)]


class MhaWeights(C.Structure):
    """b200trk_mha_weights_t"""
    _fields_ = [("in_proj_weight", C.c_void_p), ("in_proj_bias", C.c_void_p), ("out_proj_weight", C.c_void_p), ("out_proj_bias", C.c_void_p)]


class EncLayer(C.Structure):
    """b200trk_enc_layer_t"""
    _fields_ = [("self_attn", MhaWeights)] + [(n, C.c_void_p) for n in (
        "linear1_weight", "linear1_bias", "linear2_weight", "linear2_bias", "norm1_weight", "norm1_bias", "norm2_weight", "norm2_bias")]


class DecLayer(C.Structure):
    """b200trk_dec_layer_t"""
    _fields_ = [("self_attn", MhaWeights), ("cross_attn", MhaWeights)] + [(n, C.c_void_p) for n in (
        "linear1_weight", "linear1_bias", "linear2_weight", "linear2_bias", "norm1_weight", "norm1_bias", "norm2_weight", "norm2_bias",
        "norm3_weight", "norm3_bias")]


class LinearBlock(C.Structure):
    """b200trk_linear_block_t"""
    _fields_ = [(n, C.c_void_p) for n in ("weight", "bias", "bn_gamma", "bn_beta", "bn_mean", "bn_var")]


class DimpParams(C.Structure):
    """b200trk_dimp_params_t"""
    _fields_ = [("image_sample_size", C.c_int), ("search_area_scale", C.c_double), ("sample_memory_size", C.c_int),
                ("learning_rate", C.c_double), ("hard_negative_learning_rate", C.c_double), ("init_samples_minimum_weight", C.c_double),
                ("train_skipping", C.c_int), ("train_sample_interval", C.c_int), ("net_opt_iter", C.c_int),
                ("net_opt_update_iter", C.c_int), ("net_opt_hn_iter", C.c_int), ("update_classifier", C.c_int),
                ("advanced_localization", C.c_int), ("target_not_found_threshold", C.c_double), ("distractor_threshold", C.c_double),
                ("hard_negative_threshold", C.c_double), ("target_neighborhood_scale", C.c_double), ("dispalcement_scale", C.c_double),
                ("uncertain_threshold", C.c_double), ("hard_sample_threshold", C.c_double), ("target_inside_ratio", C.c_double),
                ("augmentation_expansion_factor", C.c_double), ("output_not_found_box", C.c_int),
                ("use_iou_net", C.c_int), ("iounet_k", C.c_int), ("num_init_random_boxes", C.c_int), ("box_jitter_pos", C.c_double),
                ("box_jitter_sz", C.c_double), ("maximal_aspect_ratio", C.c_double), ("box_refinement_iter", C.c_int),
                ("box_refinement_step_length", C.c_double), ("box_refinement_step_decay", C.c_double),
                ("box_refinement_relative", C.c_int), ("update_scale_when_uncertain", C.c_int),
                ("use_iounet_pos_for_learning", C.c_int), ("border_mode", C.c_int), ("patch_max_scale_change", C.c_double),
                ("score_preprocess", C.c_int), ("has_softmax_reg", C.c_int), ("softmax_reg", C.c_double)]


class CropGeom(C.Structure):
    """b200trk_crop_geom_t"""
    _fields_ = [(n, C.c_int) for n in ("df", "os_r", "os_c", "tl_r", "tl_c", "in_h", "in_w", "out_h", "out_w", "win_r", "win_c")] + \
               [("coord", C.c_float * 4), ("sample_pos", C.c_float * 2), ("sample_scale", C.c_float)]


class LocResult(C.Structure):
    """b200trk_loc_result_t"""
    _fields_ = [(n, C.c_int) for n in ("flag", "scale_ind", "r1", "c1", "r2", "c2", "use_second")] + \
               [("score1", C.c_float), ("score2", C.c_float), ("max_score", C.c_float), ("pad_", C.c_int * 6)]


class FrameInfo(C.Structure):
    """b200trk_frame_info_t"""
    _fields_ = [("bbox", C.c_float * 4), ("flag", C.c_int), ("updated", C.c_int), ("replace_ind", C.c_int), ("num_iter", C.c_int),
                ("n_stored", C.c_int), ("learning_rate", C.c_float), ("target_box", C.c_float * 4), ("max_score", C.c_float),
                ("loc", LocResult), ("crop", CropGeom), ("refined", C.c_int), ("predicted_iou", C.c_float)]


AUG_MAX = 16
AUG_KINDS = {"identity": 0, "translation": 1, "fliplr": 2, "blur": 3, "rotate": 4, "scale": 5}


class AugTransform(C.Structure):
    """b200trk_aug_transform_t"""
    _fields_ = [("kind", C.c_int), ("shift", C.c_int * 2), ("param", C.c_double * 2)]


class DimpAugment(C.Structure):
    """b200trk_dimp_augment_t"""
    _fields_ = [("num_transforms", C.c_int), ("transform", AugTransform * AUG_MAX), ("num_dropout", C.c_int),
                ("dropout_mult", C.c_void_p)]


class BatchItem(C.Structure):
    """b200trk_batch_item_t"""
    _fields_ = [("slot", C.c_int), ("image", C.c_void_p), ("H", C.c_int), ("W", C.c_int), ("init", C.c_int), ("init_bbox", C.c_double * 4)]


# name -> (restype, argtypes); every symbol of include/b200trk.h is listed (tests check the export table against it)
_VP, _I, _F = C.c_void_p, C.c_int, C.c_float
SIGNATURES = {
    "b200trk_version": (_I, []),
    "b200trk_last_error": (C.c_char_p, []),
    "b200trk_launch_count": (C.c_uint64, []),
    "b200trk_sd_last_kernel": (_I, []),
    "b200trk_debug_sd_trace": (_I, [_VP]),
    "b200trk_debug_sd_units": (_I, [_VP]),
    "b200trk_apply_filter": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP, _VP, _VP]),
    "b200trk_apply_feat_transpose": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "b200trk_conv2d_same": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "b200trk_conv1x1": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "b200trk_feature_normalize": (_I, [_VP, _I, _I, _I, _I, _F, _VP]),
    "b200trk_fourier_interp": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "b200trk_softmax_reg": (_I, [_VP, _VP, _I, _I, _I, _F, _VP]),
    "b200trk_max2d": (_I, [_VP, _I, _I, _I, _VP, _VP, _VP]),
    "b200trk_dimp_sd_gn": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _I, _F, _F, _F, _F, _F,
                                _VP, _VP, _VP]),
    "b200trk_dimp_l2_sd_gn": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _F, _F, _F, _F, _F, _F, _VP, _VP, _VP]),
    "b200trk_gn_sd_hinge": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _F, _F, _F, _I, _F, _F, _VP, _VP, _VP]),
    "b200trk_prdimp_sd_newton": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _F, _F, _F, _F, _F, _I, _F, _F,
                                      _I, _F, _F, _VP, _VP, _VP]),
    "b200trk_atom_cg_filter": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _F, _I, _I, _F, _VP]),
    "b200trk_atom_gn_joint": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _F, _F, _I, _I, _F, _VP]),
    "b200trk_eco_filter_cg": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _VP, _I, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I,
                                   _F, _F, _F, _F, _VP]),
    "b200trk_eco_joint_gn": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _VP, _F, _F, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "b200trk_eco_apply_filter": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "b200trk_eco_sample_fs": (_I, [C.POINTER(_VP), C.POINTER(_I), C.POINTER(_I), C.POINTER(_F), _I, _I, _I, _I, _VP, _VP]),
    "b200trk_eco_preprocess_sample": (_I, [_VP, C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "b200trk_eco_shift_fs": (_I, [_VP, _VP, _I, _I, _I, _I, _F, _F, _VP]),
    "b200trk_net_create": (_I, [C.POINTER(_VP), _I, C.POINTER(ConvDesc), _I, _F, _I, _I, _I, _I]),
    "b200trk_net_destroy": (_I, [_VP]),
    "b200trk_net_forward": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _VP]),
    "b200trk_net_attach_iou_head": (_I, [_VP, C.POINTER(ConvDesc)]),
    "b200trk_net_iou_from_arena": (_I, [_VP, _I, _VP, _VP, _VP]),
    "b200trk_net_iou_dims": (_I, [_VP, C.POINTER(C.c_int * 6)]),
    "b200trk_net_attach_iou_ref": (_I, [_VP, C.POINTER(ConvDesc)]),
    "b200trk_iou_modulation_create": (_I, [C.POINTER(_VP), C.POINTER(LinearBlock), C.POINTER(LinearBlock), C.POINTER(LinearBlock), _I, _I, _I, _I, _I]),
    "b200trk_iou_modulation_destroy": (_I, [_VP]),
    "b200trk_iou_modulation_dims": (_I, [_VP, C.POINTER(C.c_int * 2)]),
    "b200trk_iou_modulation_get": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "b200trk_dimp_tracker_attach_modulation_head": (_I, [_VP, _VP]),
    "b200trk_dimp_tracker_modulation": (_I, [_VP, _VP, _VP]),
    "b200trk_net_attach_filter_init": (_I, [_VP, C.POINTER(ConvDesc), _I, _I, _I]),
    "b200trk_net_filter_init_attached": (_I, [_VP]),
    "b200trk_net_filter_init": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP]),
    "b200trk_net_forward_iou": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "b200trk_net_dims": (_I, [_VP, C.POINTER(C.c_int * 9)]),
    "b200trk_net_flops": (C.c_double, [_VP]),
    "b200trk_net_num_ops": (_I, [_VP]),
    "b200trk_net_op_info": (_I, [_VP, _I, C.POINTER(C.c_int * 8)]),
    "b200trk_net_op_io": (_I, [_VP, _I, C.POINTER(C.c_int * 4)]),
    "b200trk_net_op_weights": (_I, [_VP, _I, _VP, _VP, _VP]),
    "b200trk_net_op_output": (_I, [_VP, _I, _I, _VP, _VP]),
    "b200trk_net_op_set_timing_buffer": (_I, [_VP, _I, _VP]),
    "b200trk_net_op_grid": (_I, [_VP, _I, C.POINTER(C.c_int * 4)]),
    "b200trk_net_op_splitk_reduction": (_I, [_VP, _I, C.POINTER(C.c_int)]),
    "b200trk_transformer_create": (_I, [C.POINTER(_VP), C.POINTER(EncLayer), _I, C.POINTER(DecLayer), _I, _VP, _VP, _I, _I, _I, _I, _I]),
    "b200trk_transformer_destroy": (_I, [_VP]),
    "b200trk_transformer_forward": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, _VP]),
    "b200trk_transformer_debug_num_launches": (_I, [_VP]),
    "b200trk_transformer_debug_stop_after": (_I, [_VP, _I]),
    "b200trk_transformer_debug_buffer": (_I, [_VP, _I, _VP, C.POINTER(C.c_longlong), _VP]),
    "b200trk_transformer_debug_gemm": (_I, [_VP, _I, C.POINTER(C.c_int * 15)]),
    "b200trk_tomp_tokens": (_I, [_VP] * 13 + [_I, _I, _I, _I, _I, _I, _I, _VP]),
    "b200trk_tower_create": (_I, [C.POINTER(_VP), C.POINTER(ConvDesc), _I, C.POINTER(_VP), C.POINTER(_VP), _I, _I, _I, _I, _I]),
    "b200trk_tower_destroy": (_I, [_VP]),
    "b200trk_tower_flops": (C.c_double, [_VP]),
    "b200trk_tower_forward": (_I, [_VP, _VP, _VP, _I, _VP, _VP]),
    "b200trk_tower_debug_num_launches": (_I, [_VP]),
    "b200trk_tower_debug_stop_after": (_I, [_VP, _I]),
    "b200trk_tower_debug_buffer": (_I, [_VP, _I, _I, _VP, _VP]),
    "b200trk_tower_debug_conv": (_I, [_VP, _I, C.POINTER(C.c_int * 10)]),
    "b200trk_prroi_pool_forward": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _F, _VP]),
    "b200trk_prroi_pool_backward": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _F, _VP]),
    "b200trk_prroi_pool_coor_backward": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _F, _VP]),
    "b200trk_dimp_state_create": (_I, [C.POINTER(_VP), _VP, _I, _I, _VP, _VP, _VP, _I, _F, _F, _F, _F, _F]),
    "b200trk_prdimp_state_create": (_I, [C.POINTER(_VP), _VP, _I, _I, _F, _F, _F, _F, _F, _I, _F, _F, _I, _F, _F]),
    "b200trk_dimp_state_optimizer_kind": (_I, [_VP]),
    "b200trk_dimp_state_destroy": (_I, [_VP]),
    "b200trk_dimp_state_filter": (_VP, [_VP]),
    "b200trk_dimp_state_memory_pitch": (_I, [_VP]),
    "b200trk_dimp_state_memory": (_VP, [_VP]),
    "b200trk_dimp_state_boxes": (_VP, [_VP]),
    "b200trk_dimp_state_sample_weights": (_VP, [_VP]),
    "b200trk_dimp_state_clf": (_VP, [_VP]),
    "b200trk_dimp_state_scores": (_VP, [_VP]),
    "b200trk_dimp_localize_host": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _VP]),
    "b200trk_dimp_update_host": (_I, [_VP, _I, _I, _VP, _VP, _I, _I, _VP]),
    "b200trk_iou_predictor_create": (_I, [C.POINTER(_VP), C.POINTER(LinearBlock), C.POINTER(LinearBlock), _VP, _VP, _I, _I, _I, _I, _I, _I]),
    "b200trk_iou_predictor_destroy": (_I, [_VP]),
    "b200trk_iou_predict": (_I, [_VP, _VP, _VP, _VP, _I, _I, _VP, _I, _I, _VP, _I, _VP, _VP, _VP]),
    "b200trk_iou_refine": (_I, [_VP, _VP, _VP, _VP, _I, _I, _VP, _I, _I, _VP, _I, _I, _F, _F, _I, _VP, _VP]),
    "b200trk_dimp_tracker_create": (_I, [C.POINTER(_VP), _VP, C.POINTER(DimpParams)]),
    "b200trk_dimp_tracker_destroy": (_I, [_VP]),
    "b200trk_dimp_tracker_initialize_host": (_I, [_VP, _VP, _I, _I, C.POINTER(C.c_double * 4), _VP]),
    "b200trk_augment_crops": (_I, [_VP, _I, _I, _I, _I, C.POINTER(AugTransform), _I, _VP, _VP]),
    "b200trk_dimp_tracker_init_state_augmented": (_I, [_VP, _I, _I, C.POINTER(C.c_double * 4), C.POINTER(DimpAugment), C.POINTER(CropGeom),
                                                       _VP]),
    "b200trk_dimp_tracker_initialize_augmented_host": (_I, [_VP, _VP, _I, _I, C.POINTER(C.c_double * 4), C.POINTER(DimpAugment), _VP]),
    "b200trk_dimp_tracker_init_state": (_I, [_VP, _I, _I, C.POINTER(C.c_double * 4), C.POINTER(CropGeom), C.POINTER(C.c_float * 4)]),
    "b200trk_dimp_tracker_adopt": (_I, [_VP, _I, _I, C.POINTER(C.c_float * 2), C.POINTER(C.c_float * 2), _F, C.POINTER(C.c_float * 2),
                                        _F, _F, _VP, _I, _I, _I, _I]),
    "b200trk_dimp_tracker_attach_iounet": (_I, [_VP, _VP, _VP, _VP]),
    "b200trk_dimp_tracker_set_proposal_noise": (_I, [_VP, _VP, _I]),
    "b200trk_dimp_track_host": (_I, [_VP, _VP, _I, _I, C.POINTER(FrameInfo), _VP]),
    "b200trk_dimp_track_device": (_I, [_VP, _VP, _I, _I, C.POINTER(FrameInfo), _VP]),
    "b200trk_dimp_tracker_plan_crop": (_I, [_VP, C.POINTER(CropGeom)]),
    "b200trk_dimp_tracker_commit": (_I, [_VP, C.POINTER(CropGeom), C.POINTER(LocResult), C.POINTER(FrameInfo), _VP]),
    "b200trk_dimp_tracker_commit_localize": (_I, [_VP, C.POINTER(CropGeom), C.POINTER(LocResult), C.POINTER(FrameInfo)]),
    "b200trk_dimp_tracker_proposals": (_I, [_VP, C.POINTER(CropGeom), _VP, C.POINTER(C.c_int)]),
    "b200trk_dimp_tracker_commit_refine": (_I, [_VP, C.POINTER(CropGeom), _VP, _VP, _I, C.POINTER(FrameInfo)]),
    "b200trk_dimp_tracker_commit_update": (_I, [_VP, C.POINTER(CropGeom), C.POINTER(FrameInfo), _VP]),
    "b200trk_dimp_tracker_state": (_I, [_VP, C.POINTER(C.c_float * 9)]),
    "b200trk_sample_patch": (_I, [_VP, _I, _I, C.POINTER(CropGeom), _I, _I, _VP, _VP]),
    "b200trk_dimp_localize": (_I, [_VP, _I, _I, _I, C.POINTER(DimpParams), _VP, _VP, _VP, _VP]),
    "b200trk_dimp_batch_create": (_I, [C.POINTER(_VP), _VP, _I, C.POINTER(DimpParams), _I, _VP, _VP, _VP, _I, _F, _F, _F, _F, _F]),
    "b200trk_prdimp_batch_create": (_I, [C.POINTER(_VP), _VP, _I, C.POINTER(DimpParams), _I, _F, _F, _F, _F, _F, _I, _F, _F, _I, _F, _F]),
    "b200trk_dimp_batch_destroy": (_I, [_VP]),
    "b200trk_dimp_batch_release": (_I, [_VP, _I]),
    "b200trk_dimp_batch_step_host": (_I, [_VP, C.POINTER(BatchItem), _I, C.POINTER(FrameInfo), _VP]),
    "b200trk_dimp_batch_step_device": (_I, [_VP, C.POINTER(BatchItem), _I, C.POINTER(FrameInfo), _VP]),
    "b200trk_dimp_batch_filter": (_VP, [_VP, _I]),
    "b200trk_dimp_batch_scores": (_VP, [_VP, _I]),
    "b200trk_dimp_batch_crop": (_VP, [_VP, _I]),
    "b200trk_dimp_batch_state": (_I, [_VP, _I, C.POINTER(C.c_float * 9)]),
}

_lib = None


def lib():
    """Load (once) and return the ctypes handle. Raises if the CUDA library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "pytracking_b200: %s is missing -- the CUDA extension must be built (python -c 'import "
                "__graft_entry__ as g; g.build()'); there is no CPU / PyTorch fallback." % LIB_PATH)
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)          # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(status, what=""):
    if status != 0:
        msg = lib().b200trk_last_error()
        raise RuntimeError("b200trk %s failed (status %d): %s" % (what, status, msg.decode() if msg else "?"))
