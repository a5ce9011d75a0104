"""ctypes prototypes of the U-Net entry points (include/eld_b200_unet.h)."""
import ctypes as c

vp, i32 = c.c_void_p, c.c_int


class AdamRange(c.Structure):
    """eld_adam_range"""
    _fields_ = [('offset', c.c_size_t), ('count', c.c_size_t), ('step', i32), ('lr', c.c_float), ('beta1', c.c_float),
                ('beta2', c.c_float), ('eps', c.c_float), ('weight_decay', c.c_float)]


class AdamRangeDev(c.Structure):
    """eld_adam_range_dev (step: device int*, lr: device float*)"""
    _fields_ = [('offset', c.c_size_t), ('count', c.c_size_t), ('step', vp), ('lr', vp), ('beta1', c.c_float),
                ('beta2', c.c_float), ('eps', c.c_float), ('weight_decay', c.c_float)]


AMSGRAD, MAXIMIZE, DECOUPLED = 1, 2, 4     # ELD_ADAM_*


class AdamRangeEx(c.Structure):
    """eld_adam_range_ex"""
    _fields_ = AdamRange._fields_ + [('flags', c.c_uint)]


class AdamRangeDevEx(c.Structure):
    """eld_adam_range_dev_ex (step: device int*, lr: device float*)"""
    _fields_ = AdamRangeDev._fields_ + [('flags', c.c_uint)]


def declare(lib):
    lib.eld_pack_weights.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    lib.eld_conv3x3_bf16.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32,
                                     i32, vp, i32, i32, vp]
    lib.eld_deconv2x2_bf16.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    lib.eld_deconv2x2_dgrad_bf16.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, i32, i32, i32, i32, i32,
                                             i32, vp, i32, i32, vp]
    declare_engine(lib)


def declare_engine(lib):
    f32, sz = c.c_float, c.c_size_t
    lib.eld_conv3x3_wgrad_bf16.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32, i32, vp, i32, i32, i32, vp]
    lib.eld_deconv2x2_wgrad_bf16.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32, i32, vp, i32, i32, i32, vp]
    lib.eld_unet_param_count.restype = sz
    lib.eld_unet_param_offset.argtypes = [c.c_char_p, i32, c.POINTER(sz), c.POINTER(sz)]
    lib.eld_unet_workspace_bytes.argtypes = [i32, i32, i32, i32]
    lib.eld_unet_workspace_bytes.restype = sz
    lib.eld_unet_create.argtypes = [vp, i32, i32, i32, i32, vp, sz, c.POINTER(vp)]
    lib.eld_unet_param_count_io.argtypes = [i32, i32]
    lib.eld_unet_param_count_io.restype = sz
    lib.eld_unet_param_offset_io.argtypes = [c.c_char_p, i32, i32, i32, c.POINTER(sz), c.POINTER(sz)]
    lib.eld_unet_create_io.argtypes = [vp, i32, i32, i32, i32, vp, sz, i32, i32, c.POINTER(vp)]
    lib.eld_unet_grad_buckets_io.argtypes = [i32, i32, c.POINTER(sz), i32]
    lib.eld_unet_destroy.argtypes = [vp]
    lib.eld_unet_destroy.restype = None
    lib.eld_unet_forward.argtypes = [vp, vp, vp, vp, vp]
    lib.eld_unet_train_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.eld_adam_step.argtypes = [vp, vp, vp, vp, vp, sz, f32, f32, f32, f32, f32, i32, f32, vp]
    lib.eld_unet_grad_buckets.argtypes = [c.POINTER(sz), i32]
    lib.eld_unet_bucket_events.argtypes = [vp, i32]
    lib.eld_unet_wait_bucket.argtypes = [vp, i32, vp]
    lib.eld_unet_backward.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.eld_unet_input_grad.argtypes = [vp, vp, vp, vp]
    lib.eld_unet_state_bytes.argtypes = [i32, i32, i32, i32, i32]
    lib.eld_unet_state_bytes.restype = sz
    lib.eld_unet_forward_state.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.eld_unet_backward_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.eld_unet_set_trainable.argtypes = [vp, c.POINTER(c.c_uint8), i32, i32]
    lib.eld_adam_step_segments.argtypes = [vp, vp, vp, vp, vp, c.POINTER(sz), c.POINTER(i32), i32, f32, f32, f32, f32, f32,
                                           f32, vp]
    lib.eld_adam_step_capturable.argtypes = [vp, vp, vp, vp, vp, sz, vp, vp, f32, f32, f32, f32, f32, vp]
    lib.eld_adam_step_segments_capturable.argtypes = [vp, vp, vp, vp, vp, c.POINTER(sz), c.POINTER(vp), i32, vp, f32, f32,
                                                      f32, f32, f32, vp]
    lib.eld_adam_step_ranges.argtypes = [vp, vp, vp, vp, vp, c.POINTER(AdamRange), i32, f32, vp]
    lib.eld_adam_step_ranges_capturable.argtypes = [vp, vp, vp, vp, vp, c.POINTER(AdamRangeDev), i32, f32, vp]
    lib.eld_adam_step_ranges_ex.argtypes = [vp, vp, vp, vp, vp, vp, c.POINTER(AdamRangeEx), i32, f32, vp]
    lib.eld_adam_step_ranges_ex_capturable.argtypes = [vp, vp, vp, vp, vp, vp, c.POINTER(AdamRangeDevEx), i32, f32, vp]
    lib.eld_unet_set_loss.argtypes = [vp, i32]
    lib.eld_unet_set_accumulate.argtypes = [vp, i32]
    lib.eld_clock_probe.argtypes = [vp, vp, vp]
    lib.eld_unet_profile.argtypes = [vp, i32]
    lib.eld_unet_profile_read.argtypes = [vp, i32, c.c_char_p, vp, vp, vp, c.POINTER(i32)]
    lib.eld_unet_buffer.argtypes = [vp, c.c_char_p, c.POINTER(vp), c.POINTER(i32), c.POINTER(i32)]
