"""ctypes binding of include/deephar_b200.h (libdeephar_b200.so, built in-tree by
deephar_b200/csrc/Makefile).  There is deliberately NO fallback: if the shared library
is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DEEPHAR_B200_LIB: another build of the same library (tools/: the timing-ablation build `make ABLATE=1`)
LIB_PATH = os.environ.get('DEEPHAR_B200_LIB') or os.path.join(_HERE, 'libdeephar_b200.so')


class DeepharB200Error(RuntimeError):
    pass


class dh_view(C.Structure):
    _fields_ = [('p', C.c_void_p), ('n', C.c_int32), ('h', C.c_int32), ('w', C.c_int32),
                ('c', C.c_int32), ('ld', C.c_int32)]


class dh_conv_desc(C.Structure):
    _fields_ = [('kh', C.c_int32), ('kw', C.c_int32), ('sh', C.c_int32), ('sw', C.c_int32),
                ('pad_same', C.c_int32), ('pre_relu', C.c_int32), ('post_relu', C.c_int32),
                ('n_res', C.c_int32),
                ('pre_scale', C.c_void_p), ('pre_shift', C.c_void_p),
                ('post_scale', C.c_void_p), ('post_shift', C.c_void_p),
                ('res', dh_view * 2),
                ('precision', C.c_int32), ('res_up2x', C.c_int32), ('pool_out', dh_view)]


class dh_frame_src(C.Structure):
    _fields_ = [('data', C.c_uint64), ('h', C.c_int32), ('w', C.c_int32), ('stride', C.c_int32),   # data: device pointer
                ('x0', C.c_int32), ('y0', C.c_int32), ('cw', C.c_int32), ('ch', C.c_int32), ('hflip', C.c_int32),
                ('kx_off', C.c_int32), ('ky_off', C.c_int32), ('kx_coef_off', C.c_int32), ('ky_coef_off', C.c_int32),
                ('ksx', C.c_int32), ('ksy', C.c_int32)]


class dh_frame_box(C.Structure):
    _fields_ = [('data', C.c_uint64), ('h', C.c_int32), ('w', C.c_int32), ('stride', C.c_int32),     # data: device pointer
                ('hflip', C.c_int32), ('objpos', C.c_double * 2), ('winsize', C.c_double * 2)]


# dh_prepare_frames_u8 status bits
FRAME_EMPTY, FRAME_TOO_LARGE, FRAME_BAD_BOX = 1, 2, 4


class dh_packed_w(C.Structure):
    _fields_ = [('hi', C.c_void_p), ('lo', C.c_void_p), ('cout_pad', C.c_int32), ('k', C.c_int32)]


class dh_conv_plan_info(C.Structure):
    _fields_ = [('path', C.c_int32), ('fallback', C.c_int32), ('workspace_bytes', C.c_int64),
                ('n_mtiles', C.c_int32), ('grid_x', C.c_int32), ('grid_y', C.c_int32), ('bn_cta', C.c_int32),
                ('n_kblocks', C.c_int32), ('stages', C.c_int32), ('cluster', C.c_int32), ('bm', C.c_int32),
                ('epi_tma', C.c_int32)]


class dh_clip_window(C.Structure):
    _fields_ = [('src', dh_view), ('dst', dh_view), ('ring', C.c_void_p)]


class dh_jpeg_image(C.Structure):
    _fields_ = [('data', C.c_int64), ('coef', C.c_int64 * 3), ('plane', C.c_int64 * 3), ('out', C.c_int64),
                ('h', C.c_int32), ('w', C.c_int32), ('ncomp', C.c_int32), ('hs', C.c_int32), ('vs', C.c_int32),
                ('mcus_x', C.c_int32), ('mcus_y', C.c_int32), ('bw', C.c_int32 * 3), ('bh', C.c_int32 * 3),
                ('qt', C.c_int32 * 3), ('dc', C.c_int32 * 3), ('ac', C.c_int32 * 3), ('nblocks', C.c_int32),
                ('pad', C.c_int32)]


class dh_jpeg_segment(C.Structure):
    _fields_ = [('begin', C.c_int64), ('end', C.c_int64), ('image', C.c_int32), ('mcu0', C.c_int32),
                ('mcus', C.c_int32), ('pad', C.c_int32)]


class dh_jpeg_huff(C.Structure):
    _fields_ = [('lut', C.c_uint16 * 512), ('maxcode', C.c_int32 * 18), ('valoff', C.c_int32 * 18),
                ('vals', C.c_uint8 * 256)]


class dh_jpeg_batch(C.Structure):    # pointers: device addresses
    _fields_ = [('images', C.c_uint64), ('segments', C.c_uint64), ('huff', C.c_uint64), ('qtab', C.c_uint64),
                ('data', C.c_uint64), ('coef', C.c_uint64), ('planes', C.c_uint64), ('out', C.c_uint64),
                ('status', C.c_uint64), ('coef_elems', C.c_int64), ('n_images', C.c_int32),
                ('n_segments', C.c_int32), ('max_blocks', C.c_int32), ('max_h', C.c_int32), ('max_w', C.c_int32),
                ('pad', C.c_int32)]


class dh_model_output_info(C.Structure):
    _fields_ = [('name', C.c_char * 64), ('rank', C.c_int32), ('pad', C.c_int32), ('shape', C.c_int64 * 6)]


class dh_model_info(C.Structure):
    _fields_ = [('version', C.c_int32), ('precision', C.c_int32), ('use_tensor_cores', C.c_int32),
                ('frame_items', C.c_int32), ('clip_items', C.c_int32), ('frames_per_clip', C.c_int32),
                ('input_rank', C.c_int32), ('n_outputs', C.c_int32), ('input_shape', C.c_int64 * 6),
                ('n_launches', C.c_int64), ('n_slots', C.c_int64), ('weight_bytes', C.c_int64),
                ('packed_bytes', C.c_int64), ('workspace_bytes', C.c_int64), ('activation_bytes', C.c_int64),
                ('device_bytes', C.c_int64)]


class dh_stream_info(C.Structure):
    _fields_ = [('version', C.c_int32), ('precision', C.c_int32), ('use_tensor_cores', C.c_int32),
                ('n_streams', C.c_int32), ('frames_per_clip', C.c_int32), ('input_rank', C.c_int32),
                ('input_shape', C.c_int64 * 6), ('n_frame_outputs', C.c_int32), ('n_clip_outputs', C.c_int32),
                ('n_boundary', C.c_int32), ('pad', C.c_int32), ('n_frame_launches', C.c_int64),
                ('n_clip_launches', C.c_int64), ('n_frame_slots', C.c_int64), ('n_clip_slots', C.c_int64),
                ('weight_bytes', C.c_int64), ('packed_bytes', C.c_int64), ('frame_workspace_bytes', C.c_int64),
                ('clip_workspace_bytes', C.c_int64), ('activation_bytes', C.c_int64), ('ring_bytes', C.c_int64),
                ('device_bytes', C.c_int64)]


_VP = C.POINTER(dh_view)
_DP = C.POINTER(dh_conv_desc)
_PP = C.POINTER(dh_packed_w)
_IP = C.POINTER(dh_conv_plan_info)

# name -> (restype, argtypes); every symbol declared in include/deephar_b200.h
SIGNATURES = {
    'dh_ctx_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    'dh_ctx_destroy': (C.c_int, [C.c_void_p]),
    'dh_last_error': (C.c_char_p, []),
    'dh_version': (C.c_int, []),
    'dh_launch_count': (C.c_int64, [C.c_void_p, C.c_int]),
    'dh_set_workspace': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
    'dh_set_option': (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    'dh_tc_cout_pad': (C.c_int, [C.c_int]),
    'dh_tc_k_pad': (C.c_int, [C.c_int]),
    'dh_last_conv_path': (C.c_int, [C.c_void_p]),
    'dh_fallback_count': (C.c_int64, [C.c_void_p, C.c_int]),
    'dh_comm_unique_id': (C.c_int, [C.c_void_p]),
    'dh_comm_init': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    'dh_comm_destroy': (C.c_int, [C.c_void_p]),
    'dh_allgather_f32': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    'dh_comm_info': (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    'dh_conv2d_f32': (C.c_int, [C.c_void_p, _VP, C.c_void_p, _PP, _DP, _VP, C.c_void_p]),
    'dh_sepconv2d_f32': (C.c_int, [C.c_void_p, _VP, C.c_void_p, C.c_void_p, _PP, _DP, _VP, C.c_void_p]),
    'dh_conv2d_plan': (C.c_int, [C.c_void_p, _VP, C.c_void_p, _PP, _DP, _VP, _IP]),
    'dh_sepconv2d_plan': (C.c_int, [C.c_void_p, _VP, C.c_void_p, C.c_void_p, _PP, _DP, _VP, _IP]),
    'dh_maxpool2d_f32': (C.c_int, [C.c_void_p, _VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _VP, C.c_void_p]),
    'dh_upsample2x_add_f32': (C.c_int, [C.c_void_p, _VP, _VP, _VP, C.c_void_p]),
    'dh_add_n_f32': (C.c_int, [C.c_void_p, _VP, C.c_int, C.c_void_p, C.c_void_p, C.c_int, _VP, C.c_void_p]),
    'dh_softargmax2d_f32': (C.c_int, [C.c_void_p, _VP, _VP, C.c_float, C.c_int, C.c_void_p, C.c_void_p, _VP, C.c_void_p]),
    'dh_softargmax2d_ctx_f32': (C.c_int, [C.c_void_p, _VP, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    'dh_softargmax3d_f32': (C.c_int, [C.c_void_p, _VP, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    'dh_softargmax3d_ex_f32': (C.c_int, [C.c_void_p, _VP, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, _VP, C.c_void_p]),
    'dh_crop_resize_norm_u8': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'dh_prepare_frames_workspace': (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    'dh_prepare_frames_u8': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'dh_jpeg_decode': (C.c_int, [C.c_void_p, C.POINTER(dh_jpeg_batch), C.c_int, C.c_void_p]),
    'dh_pose_eval_f64': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'dh_pose_to_image_f32': (C.c_int, [C.c_void_p, _VP, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    'dh_kron_pool_f32': (C.c_int, [C.c_void_p, _VP, _VP, C.c_void_p, C.c_void_p]),
    'dh_zeropad2d_f32': (C.c_int, [C.c_void_p, _VP, C.c_int, C.c_int, _VP, C.c_void_p]),
    'dh_maxmin_pool2d_f32': (C.c_int, [C.c_void_p, _VP, _VP, C.c_void_p]),
    'dh_global_maxmin_softmax_f32': (C.c_int, [C.c_void_p, _VP, C.c_void_p, C.c_void_p]),
    'dh_mask_mul_f32': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    'dh_clip_window_f32': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    'dh_model_inspect': (C.c_int, [C.c_char_p, C.POINTER(dh_model_info), C.POINTER(C.c_int64), C.c_int,
                                   C.POINTER(dh_model_output_info), C.c_int]),
    'dh_model_load': (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    'dh_model_set_batch': (C.c_int, [C.c_void_p, C.c_int]),
    'dh_model_batch': (C.c_int, [C.c_void_p]),
    'dh_model_input': (C.c_int, [C.c_void_p, _VP]),
    'dh_model_forward': (C.c_int, [C.c_void_p, C.c_void_p]),
    'dh_model_output': (C.c_int, [C.c_void_p, C.c_int, _VP, C.POINTER(dh_model_output_info)]),
    'dh_model_free': (C.c_int, [C.c_void_p]),
    'dh_stream_ready_f32': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                      C.c_void_p]),
    'dh_stream_inspect': (C.c_int, [C.c_char_p, C.POINTER(dh_stream_info), C.POINTER(dh_model_output_info), C.c_int]),
    'dh_stream_load': (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    'dh_stream_input': (C.c_int, [C.c_void_p, _VP]),
    'dh_stream_push': (C.c_int, [C.c_void_p, C.c_void_p]),
    'dh_stream_reset': (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_void_p]),
    'dh_stream_output': (C.c_int, [C.c_void_p, C.c_int, _VP, C.POINTER(dh_model_output_info)]),
    'dh_stream_ready': (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    'dh_stream_free': (C.c_int, [C.c_void_p]),
}

_lib = None


def lib():
    """Load the shared library (once) and bind every declared symbol."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DeepharB200Error(
                '%s not found: build it with `make -C deephar_b200/csrc` (or '
                '`python -c "import __graft_entry__ as g; g.build()"`). There is no CPU fallback.'
                % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, what=''):
    if rc != 0:
        msg = lib().dh_last_error()
        raise DeepharB200Error('%s failed (rc=%d): %s' % (what, rc, msg.decode() if msg else ''))


def view(ptr, n, h, w, c, ld=None):
    return dh_view(ptr, n, h, w, c, c if ld is None else ld)


class Context(object):
    def __init__(self, device=0):
        self.handle = C.c_void_p()
        check(lib().dh_ctx_create(C.byref(self.handle), device), 'dh_ctx_create')

    def launch_count(self, reset=False):
        return int(lib().dh_launch_count(self.handle, 1 if reset else 0))

    def set_workspace(self, ptr, nbytes):
        check(lib().dh_set_workspace(self.handle, ptr, nbytes), 'dh_set_workspace')

    def __del__(self):
        try:
            if self.handle:
                lib().dh_ctx_destroy(self.handle)
        except Exception:
            pass
