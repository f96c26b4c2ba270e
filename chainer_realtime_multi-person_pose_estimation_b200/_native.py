"""ctypes binding of libopb.so (C ABI: include/opb.h).  Fails loudly when the CUDA library
is missing or no H100 is present -- there is no CPU fallback in this package."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OPB_LIB_PATH", os.path.join(HERE, "libopb.so"))   # OPB_LIB_PATH: A/B builds only

OPB_HOST, OPB_DEVICE = 0, 1
F32_NCHW, U8_NHWC_BGR = 0, 1
PRECISION_FAST, PRECISION_PARITY, PRECISION_COMP = 0, 1, 2
UPSAMPLE_BILINEAR_AC, UPSAMPLE_BICUBIC = 0, 1
ERR_CUDA, ERR_ARG, ERR_STATE, ERR_CAPACITY, ERR_INDEX, ERR_UNSUPPORTED = -1, -2, -3, -4, -5, -6
N_JOINTS, N_LIMBS, MAX_TAPS = 18, 19, 64


class OpbParams(C.Structure):
    _fields_ = [("limbs", (C.c_int32 * 2) * N_LIMBS),
                ("heatmap_peak_thresh", C.c_double), ("inner_product_thresh", C.c_double),
                ("limb_length_ratio", C.c_double), ("length_penalty_value", C.c_double),
                ("n_subset_limbs_thresh", C.c_double), ("subset_score_thresh", C.c_double),
                ("n_integ_points", C.c_int32), ("n_integ_points_thresh", C.c_int32),
                ("gauss_radius", C.c_int32), ("reserved0", C.c_int32),
                ("gauss_taps", C.c_double * MAX_TAPS),
                ("max_peaks", C.c_int32), ("max_candidates", C.c_int32), ("max_persons", C.c_int32),
                ("reserved1", C.c_int32)]


PERSON_DTYPE = np.dtype([("score", "<f8"), ("count", "<f8"), ("peak_id", "<i4", (N_JOINTS,)),
                         ("x", "<i4", (N_JOINTS,)), ("y", "<i4", (N_JOINTS,)), ("pad", "<i4", (2,))])
HEADER_DTYPE = np.dtype([("n_peaks", "<i4"), ("n_persons", "<i4"), ("status", "<i4"), ("n_connections", "<i4")])
CROP_DTYPE = np.dtype([("left", "<i4"), ("top", "<i4"), ("right", "<i4"), ("bottom", "<i4"), ("flip", "<i4"),
                       ("reserved", "<i4")])      # opb_crop
PART_DTYPE = np.dtype([("kind", "<i4"), ("left", "<i4"), ("top", "<i4"), ("right", "<i4"), ("bottom", "<i4"),
                       ("first_point", "<i4")])   # opb_part
PART_FACE, PART_HAND = 0, 1
WB_PART_DTYPE = np.dtype([("kind", "<i4"), ("left", "<i4"), ("top", "<i4"), ("right", "<i4"), ("bottom", "<i4"),
                          ("row", "<i4"), ("person", "<i4"), ("side", "<i4")])   # opb_wb_part
SIDE_FACE, SIDE_LEFT, SIDE_RIGHT = 0, 1, 2
PART_POINTS = {PART_FACE: 70, PART_HAND: 21}
assert PERSON_DTYPE.itemsize == 240 and HEADER_DTYPE.itemsize == 16 and CROP_DTYPE.itemsize == 24
assert PART_DTYPE.itemsize == 24 and WB_PART_DTYPE.itemsize == 32
CONV_PROBLEM_DTYPE = np.dtype([(f, "<i4") for f in (
    "in_h", "in_w", "in_c", "in_ctot", "in_coff", "out_h", "out_w", "out_c", "out_ctot", "out_coff", "cout_valid", "relu",
    "pool", "has_out32", "cin_pad", "cout_pad")] + [("acc_scale", "<f4"), ("reserved", "<i4")])    # opb_conv_problem
CONV_RECORD_DTYPE = np.dtype([("tag", "S32"), ("wkey", "S48", (2,))] + [(f, "<i4") for f in (
    "ks", "bn", "drain", "comp", "n_problems", "grid", "shared_in", "reserved")] + [
    ("prob", CONV_PROBLEM_DTYPE, (2,))])                                                              # opb_conv_record
assert CONV_PROBLEM_DTYPE.itemsize == 72 and CONV_RECORD_DTYPE.itemsize == 304
KP_STAGE_CROP_DTYPE = np.dtype([(f, "<i4") for f in (
    "left", "top", "right", "bottom", "flip", "frame", "vh", "vw")])                                 # opb_kp_stage_crop
CHANNEL_MAX_DTYPE = np.dtype([("value", "<f4"), ("count", "<i4"), ("key0", "<i4"), ("key1", "<i4")])  # opb_channel_max
assert KP_STAGE_CROP_DTYPE.itemsize == 32 and CHANNEL_MAX_DTYPE.itemsize == 16


def crop_table(bboxes, flips=None):
    """(left, top, right, bottom) integer boxes (+ per-box flip flags) -> opb_crop array.  ValueError for a box that is
    not four integers or whose canvas (bottom-top) x (right-left) is empty, so that nothing is launched for it."""
    bboxes = list(bboxes)
    flips = [False] * len(bboxes) if flips is None else list(flips)
    if len(flips) != len(bboxes):
        raise ValueError("%d boxes but %d flip flags" % (len(bboxes), len(flips)))
    table = np.zeros(len(bboxes), CROP_DTYPE)
    lim = np.iinfo(np.int32)
    for i, (b, f) in enumerate(zip(bboxes, flips)):
        try:
            vals = tuple(b)
        except TypeError:
            raise ValueError("bbox %d is not a (left, top, right, bottom) tuple: %r" % (i, b))
        if len(vals) != 4 or not all(isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
                                     for v in vals):
            raise ValueError("bbox %d must be four integers (left, top, right, bottom): %r" % (i, b))
        left, top, right, bottom = (int(v) for v in vals)
        if not all(lim.min <= v <= lim.max for v in (left, top, right, bottom)):
            raise ValueError("bbox %d does not fit int32: %r" % (i, b))
        if right - left <= 0 or bottom - top <= 0:
            raise ValueError("bbox %d gives an empty crop (%d x %d): %r" % (i, bottom - top, right - left, b))
        table[i] = (left, top, right, bottom, int(bool(f)), 0)
    return table

_SIGNATURES = {
    "opb_version": (C.c_int, []),
    "opb_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(OpbParams)]),
    "opb_destroy": (None, [C.c_void_p]),
    "opb_last_error": (C.c_char_p, [C.c_void_p]),
    "opb_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "opb_synchronize": (C.c_int, [C.c_void_p]),
    "opb_load_weights": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "opb_finalize_weights": (C.c_int, [C.c_void_p, C.c_int]),
    "opb_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                              C.c_void_p, C.c_int]),
    "opb_upsample": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                               C.c_int, C.c_int, C.c_int]),
    "opb_peaks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                            C.POINTER(C.c_int)]),
    "opb_connections": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                  C.c_double, C.c_void_p, C.c_int, C.c_void_p]),
    "opb_candidates": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                 C.c_double, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "opb_group": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                            C.POINTER(C.c_int)]),
    "opb_detect_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "opb_postprocess_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int]),
    "opb_resize_linear_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                       C.c_int, C.c_int]),
    "opb_resize_cubic_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                      C.c_int, C.c_int]),
    "opb_precise_add_scale_orig": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_void_p, C.c_int, C.c_int]),
    "opb_detect_image": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_double, C.c_void_p, C.c_void_p, C.c_int]),
    "opb_draw_person_pose": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_int]),
    "opb_draw_last_result": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double,
                                       C.c_void_p, C.c_int]),
    "opb_draw_whole_body": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "opb_stream_submit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int]),
    "opb_stream_collect": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "opb_stream_join": (C.c_int, [C.c_void_p]),
    "opb_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "opb_nccl_comm_init": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p]),
    "opb_nccl_comm_destroy": (C.c_int, [C.c_void_p]),
    "opb_record_block_bytes": (C.c_size_t, [C.c_void_p, C.c_int]),
    "opb_allgather_results": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "opb_keypoints_detect": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "opb_keypoints_from_heatmaps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                              C.c_double, C.c_void_p, C.c_void_p]),
    "opb_keypoints_detect_crops": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                             C.c_int, C.c_double, C.c_void_p, C.c_void_p]),
    "opb_precise_add_scale_unpadded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                 C.c_int, C.c_int]),
    "opb_get_image_detail": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_void_p,
                                       C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "opb_precise_begin": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "opb_precise_add_scale": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_int, C.c_int]),
    "opb_precise_finish": (C.c_int, [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_int]),
    "opb_download_maps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "opb_device_buffer": (C.c_void_p, [C.c_void_p, C.c_int]),
    "opb_launch_count": (C.c_int64, [C.c_void_p]),
    "opb_time_stage": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_float)]),
    "opb_test_conv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "opb_test_conv_first": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "opb_test_chain_convs": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "opb_test_chain_conv_run": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "opb_test_keypoint_stages": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_size_t,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                           C.c_void_p, C.c_void_p, C.c_void_p]),
    "opb_cascade_load": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "opb_cascade_detect": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int,
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "opb_face_detect_frame": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int,
                                        C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, C.c_void_p, C.c_int,
                                        C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p]),
    "opb_test_cascade_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
                                           C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                           C.POINTER(C.c_int)]),
    "opb_whole_body_frame": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_double, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                       C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "opb_test_whole_body_boxes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    "opb_whole_body_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_double, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                       C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "opb_test_whole_body_boxes_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double,
                                                  C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p]),
}

_lib = None


def load_library():
    """dlopen libopb.so and declare every symbol of include/opb.h (no GPU needed for this)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError("libopb.so is missing (%s). Build it with `python __graft_entry__.py build` "
                           "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def exported_symbols():
    return sorted(_SIGNATURES)


def _ptr(a):
    return None if a is None else C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else int(a))


class OpbError(RuntimeError):
    pass


class Engine(object):
    """One device context (opb_ctx) + the weights of one CocoPoseNet."""

    def __init__(self, device, params, precision=PRECISION_COMP):
        self.lib = load_library()
        self.ctx = C.c_void_p()
        self.params = params
        self.max_peaks, self.max_persons = params.max_peaks, params.max_persons
        rc = self.lib.opb_create(C.byref(self.ctx), int(device), C.byref(params))
        if rc != 0:
            msg = self.lib.opb_last_error(None)
            self.ctx = None
            raise OpbError("opb_create failed (%d): %s" % (rc, msg.decode() if msg else "?"))
        self.precision = precision
        self.device = int(device)
        self._weights_ready = False

    def __del__(self):
        try:
            if getattr(self, "ctx", None):
                self.lib.opb_destroy(self.ctx)
                self.ctx = None
        except Exception:
            pass

    def _check(self, rc):
        if rc == 0:
            return
        msg = self.lib.opb_last_error(self.ctx)
        msg = msg.decode() if msg else ""
        if rc == ERR_INDEX:
            raise IndexError(msg or "list assignment index out of range")   # pose_detector.py:197
        raise OpbError("libopb error %d: %s" % (rc, msg))

    def raise_for_status(self, status):
        if status == 0:
            return
        if status == ERR_INDEX:
            raise IndexError("list assignment index out of range")
        raise OpbError("device post-process status %d (capacity exceeded: raise max_peaks / max_candidates / "
                       "max_persons)" % status)

    # -- weights ---------------------------------------------------------------------------
    def load_model(self, model, precision=None):
        """model: object with children_items() -> (name, link with .W.data/.b.data)."""
        if precision is not None:
            self.precision = precision
        for name, link in model.children_items():
            W = np.ascontiguousarray(link.W.data, np.float32)
            b = np.ascontiguousarray(link.b.data, np.float32)
            shape = (C.c_int64 * 4)(*W.shape)
            self._check(self.lib.opb_load_weights(self.ctx, name.encode(), _ptr(W), shape, _ptr(b)))
        self._check(self.lib.opb_finalize_weights(self.ctx, int(self.precision)))
        self._weights_ready = True
        last = dict(model.children_items()).get("conv6_2_CPM")      # FaceNet / HandNet: channels of the final maps
        self.kp_channels = int(last.W.data.shape[0]) if last is not None else 0

    def set_stream(self, stream_handle):
        self._check(self.lib.opb_set_stream(self.ctx, C.c_void_p(int(stream_handle) if stream_handle else 0)))

    def synchronize(self):
        self._check(self.lib.opb_synchronize(self.ctx))

    # -- forward ----------------------------------------------------------------------------
    def forward(self, x):
        """x: [N,3,H,W] float32 (preprocessed) or [N,H,W,3] uint8 BGR.  Returns numpy
        (paf [N,38,h,w], heat [N,19,h,w])."""
        x = np.ascontiguousarray(x)
        if x.dtype == np.uint8:
            n, h, w, _ = x.shape
            fmt = U8_NHWC_BGR
        else:
            x = np.ascontiguousarray(x, np.float32)
            n, _, h, w = x.shape
            fmt = F32_NCHW
        paf = np.empty((n, 38, h // 8, w // 8), np.float32)
        heat = np.empty((n, 19, h // 8, w // 8), np.float32)
        self._check(self.lib.opb_forward(self.ctx, _ptr(x), fmt, OPB_HOST, n, h, w, _ptr(paf), _ptr(heat), OPB_HOST))
        return paf, heat

    def upsample(self, maps, out_h, out_w, mode=UPSAMPLE_BILINEAR_AC):
        maps = np.ascontiguousarray(maps, np.float32)
        lead = maps.shape[:-2]
        h, w = maps.shape[-2:]
        planes = int(np.prod(lead)) if lead else 1
        out = np.empty(lead + (out_h, out_w), np.float32)
        self._check(self.lib.opb_upsample(self.ctx, mode, _ptr(maps), OPB_HOST, planes, h, w, _ptr(out), OPB_HOST,
                                          out_h, out_w))
        return out

    # -- stage methods ------------------------------------------------------------------------
    def peaks(self, heatmaps):
        hm = np.ascontiguousarray(heatmaps, np.float32)
        c1, h, w = hm.shape
        out = np.empty((self.max_peaks, 5), np.float64)
        n = C.c_int(0)
        self._check(self.lib.opb_peaks(self.ctx, _ptr(hm), OPB_HOST, c1, h, w, _ptr(out), self.max_peaks, C.byref(n)))
        return out[:n.value].copy()

    def connections(self, pafs, all_peaks, img_len):
        pafs = np.ascontiguousarray(pafs, np.float32)
        _, h, w = pafs.shape
        pk = np.ascontiguousarray(all_peaks, np.float64).reshape(-1, 5)
        cap = max(len(pk), 1) * 2
        out = np.empty((cap, 3), np.float64)
        counts = np.zeros(N_LIMBS, np.int32)
        self._check(self.lib.opb_connections(self.ctx, _ptr(pafs), OPB_HOST, h, w, _ptr(pk), len(pk), float(img_len),
                                             _ptr(out), cap, _ptr(counts)))
        res, o = [], 0
        for c in counts:
            res.append(out[o:o + c].copy() if c else np.zeros((0, 3)))
            o += int(c)
        return res

    def candidates(self, paf, cand_a, cand_b, img_len):
        paf = np.ascontiguousarray(paf, np.float32)
        _, h, w = paf.shape
        a = np.ascontiguousarray(cand_a, np.float64).reshape(-1, 4)
        b = np.ascontiguousarray(cand_b, np.float64).reshape(-1, 4)
        cap = max(len(a) * len(b), 1)
        out = np.empty((cap, 3), np.float64)
        n = C.c_int(0)
        self._check(self.lib.opb_candidates(self.ctx, _ptr(paf), h, w, _ptr(a), len(a), _ptr(b), len(b), float(img_len),
                                            _ptr(out), cap, C.byref(n)))
        return out[:n.value].copy()

    def group(self, all_connections, peaks):
        pk = np.ascontiguousarray(peaks, np.float64).reshape(-1, 5)
        counts = np.array([len(c) for c in all_connections], np.int32)
        flat = (np.concatenate([np.asarray(c, np.float64).reshape(-1, 3) for c in all_connections], axis=0)
                if counts.sum() else np.zeros((0, 3)))
        flat = np.ascontiguousarray(flat[:, :3], np.float64)
        out = np.empty((self.max_persons, 20), np.float64)
        n = C.c_int(0)
        self._check(self.lib.opb_group(self.ctx, _ptr(flat), _ptr(counts), _ptr(pk), len(pk), _ptr(out),
                                       self.max_persons, C.byref(n)))
        return out[:n.value].copy()

    # -- fused batch path -------------------------------------------------------------------
    def detect_batch(self, imgs, map_h, map_w, img_len=None, inject_paf=None, inject_heat=None, imgs_ptr=None,
                     headers=None, persons=None):
        """imgs: [N,H,W,3] uint8 BGR (network-input size) host array, or a device pointer via
        imgs_ptr=(ptr, n, h, w).  inject_*: device pointers (ints) or None."""
        if imgs_ptr is not None:
            ptr, n, h, w = imgs_ptr
            src, loc = C.c_void_p(int(ptr)), OPB_DEVICE
        else:
            imgs = np.ascontiguousarray(imgs, np.uint8)
            n, h, w, _ = imgs.shape
            src, loc = _ptr(imgs), OPB_HOST
        if headers is None:
            headers = np.empty(n, HEADER_DTYPE)
        if persons is None:
            persons = np.empty((n, self.max_persons), PERSON_DTYPE)
        self._check(self.lib.opb_detect_batch(self.ctx, src, loc, n, h, w, map_h, map_w,
                                              float(map_w if img_len is None else img_len),
                                              C.c_void_p(int(inject_paf)) if inject_paf else None,
                                              C.c_void_p(int(inject_heat)) if inject_heat else None,
                                              _ptr(headers), _ptr(persons), OPB_HOST))
        return headers, persons

    def postprocess_batch(self, paf_lo, heat_lo, map_h, map_w, img_len=None):
        """Network outputs paf_lo [N,38,h8,w8] / heat_lo [N,19,h8,w8] float32 (host) -> (headers[N],
        persons[N, max_persons]): upsample, peaks, connections, grouping (opb_postprocess_batch)."""
        paf_lo = np.ascontiguousarray(paf_lo, np.float32)
        heat_lo = np.ascontiguousarray(heat_lo, np.float32)
        n, _, h8, w8 = paf_lo.shape
        assert paf_lo.shape[1] == 38 and heat_lo.shape == (n, 19, h8, w8)
        headers = np.empty(n, HEADER_DTYPE)
        persons = np.empty((n, self.max_persons), PERSON_DTYPE)
        self._check(self.lib.opb_postprocess_batch(self.ctx, _ptr(paf_lo), _ptr(heat_lo), OPB_HOST, n, h8, w8, map_h, map_w,
                                                   float(map_w if img_len is None else img_len), _ptr(headers),
                                                   _ptr(persons), OPB_HOST))
        return headers, persons

    def resize_linear_u8(self, imgs, out_h, out_w):
        """cv2.resize(img, (out_w, out_h)) (INTER_LINEAR, uint8) on the device; imgs [N,H,W,3] or [H,W,3]."""
        a = np.ascontiguousarray(imgs, np.uint8)
        single = a.ndim == 3
        if single:
            a = a[None]
        n, h0, w0, _ = a.shape
        out = np.empty((n, out_h, out_w, 3), np.uint8)
        self._check(self.lib.opb_resize_linear_u8(self.ctx, _ptr(a), OPB_HOST, n, h0, w0, _ptr(out), OPB_HOST, out_h, out_w))
        return out[0] if single else out

    def resize_cubic_u8(self, imgs, out_h, out_w):
        """cv2.resize(img, (out_w, out_h), interpolation=cv2.INTER_CUBIC) (uint8, OpenCV's own non-IPP path) on the
        device; imgs [N,H,W,3] or [H,W,3]."""
        a = np.ascontiguousarray(imgs, np.uint8)
        single = a.ndim == 3
        if single:
            a = a[None]
        n, h0, w0, _ = a.shape
        out = np.empty((n, out_h, out_w, 3), np.uint8)
        self._check(self.lib.opb_resize_cubic_u8(self.ctx, _ptr(a), OPB_HOST, n, h0, w0, _ptr(out), OPB_HOST, out_h, out_w))
        return out[0] if single else out

    def draw_person_pose(self, img, poses):
        """draw_person_pose(orig_img, poses) (pose_detector.py:520-553) on the device; poses float [P,18,3]."""
        a = np.ascontiguousarray(img, np.uint8)
        h, w, _ = a.shape
        ip = np.ascontiguousarray(np.asarray(poses).round().astype('i').reshape(-1, 18, 3), np.int32)
        out = np.empty_like(a)
        self._check(self.lib.opb_draw_person_pose(self.ctx, _ptr(a), OPB_HOST, h, w, _ptr(ip) if len(ip) else None, len(ip),
                                                  _ptr(out), OPB_HOST))
        return out

    def draw_last_result(self, img, sx, sy, image_index=0):
        """Overlay of the persons of the last detect call, taken from the device-resident records."""
        a = np.ascontiguousarray(img, np.uint8)
        h, w, _ = a.shape
        out = np.empty_like(a)
        self._check(self.lib.opb_draw_last_result(self.ctx, int(image_index), _ptr(a), OPB_HOST, h, w, float(sx), float(sy),
                                                  _ptr(out), OPB_HOST))
        return out

    def draw_whole_body(self, img, poses, parts):
        """The whole-body picture of demo.py:28-57 on the device (opb_draw_whole_body): poses float [P,18,3] as for
        draw_person_pose; parts (kind, bbox, keypoints) with kind PART_FACE / PART_HAND, bbox (left, top, right, bottom)
        and keypoints the [x, y, conf] / None list of the detectors, in crop coordinates."""
        a = np.ascontiguousarray(img, np.uint8)
        h, w, _ = a.shape
        ip = np.ascontiguousarray(np.asarray(poses).round().astype('i').reshape(-1, 18, 3), np.int32)
        table = np.zeros(len(parts), PART_DTYPE)
        rows = []
        for i, (kind, bbox, kps) in enumerate(parts):
            table[i] = (kind,) + tuple(int(v) for v in bbox) + (len(rows),)
            rows.extend((int(k[0]), int(k[1]), 1) if k else (0, 0, 0) for k in kps)
        pts = np.array(rows, np.int64).reshape(-1, 3)
        lim = np.iinfo(np.int32)
        if pts.size and (pts.min() < lim.min or pts.max() > lim.max):
            raise ValueError("a keypoint coordinate does not fit int32")
        pts = np.ascontiguousarray(pts, np.int32)
        out = np.empty_like(a)
        self._check(self.lib.opb_draw_whole_body(self.ctx, _ptr(a), OPB_HOST, h, w, _ptr(ip) if len(ip) else None, len(ip),
                                                 _ptr(table) if len(table) else None, len(table),
                                                 _ptr(pts) if len(pts) else None, len(pts), _ptr(out), OPB_HOST))
        return out

    def detect_image(self, img, in_h, in_w, map_h, map_w, img_len=None):
        """One BGR frame of any size: upload, device resize, full pipeline (opb_detect_image)."""
        img = np.ascontiguousarray(img, np.uint8)
        oh, ow, _ = img.shape
        headers = np.empty(1, HEADER_DTYPE)
        persons = np.empty((1, self.max_persons), PERSON_DTYPE)
        self._check(self.lib.opb_detect_image(self.ctx, _ptr(img), OPB_HOST, oh, ow, in_h, in_w, map_h, map_w,
                                              float(map_w if img_len is None else img_len), _ptr(headers),
                                              _ptr(persons), OPB_HOST))
        return headers, persons

    def stream_submit(self, frames, in_h, in_w, map_h, map_w, slot, img_len=None, inject_paf=None, inject_heat=None,
                      device=False):
        """Enqueue one batch [N,H0,W0,3] uint8 on `slot` (0/1) without waiting (opb_stream_submit).  `frames`: a
        NumPy array (host), or (address, n, h, w) of a pinned host buffer -- or of a device buffer with device=True."""
        if isinstance(frames, np.ndarray):
            frames = np.ascontiguousarray(frames, np.uint8)
            if frames.ndim == 3:
                frames = frames[None]
            n, oh, ow, _ = frames.shape
            ptr = _ptr(frames)
            self._stream_keep = getattr(self, "_stream_keep", {})
            self._stream_keep[slot] = frames          # pinned buffers are read asynchronously: keep them alive
        else:                                         # (data_ptr, n, h, w) of a pinned buffer owned by the caller
            addr, n, oh, ow = frames
            ptr = C.c_void_p(addr)
        self._stream_n = getattr(self, "_stream_n", {})
        self._stream_n[slot] = n
        self._check(self.lib.opb_stream_submit(self.ctx, ptr, OPB_DEVICE if device else OPB_HOST, n, oh, ow, in_h, in_w,
                                               map_h, map_w,
                                               float(map_w if img_len is None else img_len),
                                               C.c_void_p(inject_paf or 0), C.c_void_p(inject_heat or 0), slot))

    # ---- multi-GPU: the ONE collective of the path (include/opb.h: opb_allgather_results)
    def nccl_unique_id(self):
        """128-byte NCCL id (rank 0 creates it and ships it to the other ranks, e.g. torch.distributed.broadcast)."""
        buf = np.zeros(128, np.uint8)
        rc = self.lib.opb_nccl_unique_id(C.c_void_p(buf.ctypes.data))
        if rc:
            raise OpbError("opb_nccl_unique_id failed (%d): %s" % (rc, (self.lib.opb_last_error(None) or b"").decode()))
        return buf

    def nccl_comm_init(self, world, rank, unique_id):
        comm = C.c_void_p()
        uid = np.ascontiguousarray(unique_id, np.uint8)
        self._check(self.lib.opb_nccl_comm_init(self.ctx, C.byref(comm), int(world), int(rank), C.c_void_p(uid.ctypes.data)))
        self._nccl_comm = comm
        return comm

    def record_block_bytes(self, n):
        return int(self.lib.opb_record_block_bytes(self.ctx, int(n)))

    def allgather_results(self, slot, gathered_dev_ptr, comm=None):
        """ncclAllGather of streaming slot `slot`'s device-resident record block into the device buffer at
        gathered_dev_ptr (world x record_block_bytes(n) bytes), on the slot's stream behind its pipeline."""
        self._check(self.lib.opb_allgather_results(self.ctx, comm if comm is not None else self._nccl_comm, int(slot),
                                                   C.c_void_p(int(gathered_dev_ptr))))

    def stream_join(self):
        """Make the context's stream wait for every submitted, uncollected batch (opb_stream_join)."""
        self._check(self.lib.opb_stream_join(self.ctx))

    def stream_collect(self, slot):
        """Block until the batch submitted on `slot` is done; returns (headers[N], persons[N, max_persons])."""
        n = self._stream_n[slot]
        headers = np.empty(n, HEADER_DTYPE)
        persons = np.empty((n, self.max_persons), PERSON_DTYPE)
        self._check(self.lib.opb_stream_collect(self.ctx, slot, _ptr(headers), _ptr(persons)))
        return headers, persons

    # -- face / hand nets (include/opb.h: opb_keypoints_*) ---------------------------------------
    def forward_keypoint_maps(self, x, n_out=None):
        """FaceNet / HandNet forward: x [N,3,H,W] float32 (already /256 - 0.5) or [N,H,W,3] uint8 -> [N,C,h,w]."""
        x = np.ascontiguousarray(x)
        if x.dtype == np.uint8:
            n, h, w, _ = x.shape
            fmt = U8_NHWC_BGR
        else:
            x = np.ascontiguousarray(x, np.float32)
            n, _, h, w = x.shape
            fmt = F32_NCHW
        heat = np.empty((n, n_out or self.kp_channels, h // 8, w // 8), np.float32)
        self._check(self.lib.opb_forward(self.ctx, _ptr(x), fmt, OPB_HOST, n, h, w, None, _ptr(heat), OPB_HOST))
        return heat

    @staticmethod
    def _keypoint_list(out, valid):
        return [[int(x), int(y), np.float32(c)] if v else None for (x, y, c), v in zip(out, valid)]

    def keypoints_detect(self, img, net_size, thresh, mirror=False, return_maps=False):
        """One BGR crop -> list of [x, y, conf] / None per keypoint channel (opb_keypoints_detect)."""
        img = np.ascontiguousarray(img, np.uint8)
        h, w, _ = img.shape
        planes = self.kp_channels - 1
        out = np.empty((planes, 3), np.float64)
        valid = np.empty(planes, np.int32)
        maps = np.empty((planes, h, w), np.float32) if return_maps else None
        self._check(self.lib.opb_keypoints_detect(self.ctx, _ptr(img), OPB_HOST, h, w, net_size, int(bool(mirror)),
                                                  float(thresh), _ptr(out), _ptr(valid),
                                                  _ptr(maps) if return_maps else None))
        kps = self._keypoint_list(out, valid)
        return (kps, maps) if return_maps else kps

    def keypoints_detect_crops(self, frame, crops, net_size, thresh):
        """All crops of one BGR frame [H,W,3] -> one keypoint list per crop (opb_keypoints_detect_crops).  `crops`: an
        opb_crop array (crop_table) or (left, top, right, bottom[, flip]) tuples; crop i gives what keypoints_detect
        gives for flip_i(crop_image(frame, bbox_i)) with mirror=flip_i."""
        frame = np.asarray(frame)
        if frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be a uint8 [H, W, 3] image, got %s %s" % (frame.dtype, frame.shape))
        frame = np.ascontiguousarray(frame)
        if not (isinstance(crops, np.ndarray) and crops.dtype == CROP_DTYPE):
            crops = list(crops)
            crops = crop_table([c[:4] for c in crops], [len(c) > 4 and bool(c[4]) for c in crops])
        crops = np.ascontiguousarray(crops)
        n = len(crops)
        planes = max(self.kp_channels - 1, 0)      # 0 on a pose context, which the library refuses (OPB_ERR_STATE)
        out = np.empty((n, planes, 3), np.float64)
        valid = np.empty((n, planes), np.int32)
        h, w, _ = frame.shape
        self._check(self.lib.opb_keypoints_detect_crops(self.ctx, _ptr(frame), OPB_HOST, h, w, _ptr(crops), n,
                                                        int(net_size), float(thresh), _ptr(out), _ptr(valid)))
        return [self._keypoint_list(o, v) for o, v in zip(out, valid)]

    def keypoints_from_heatmaps(self, heatmaps, thresh, mirror=False):
        """heatmaps [C,H,W] float32, background channel already dropped (opb_keypoints_from_heatmaps)."""
        hm = np.ascontiguousarray(heatmaps, np.float32)
        planes, h, w = hm.shape
        out = np.empty((planes, 3), np.float64)
        valid = np.empty(planes, np.int32)
        self._check(self.lib.opb_keypoints_from_heatmaps(self.ctx, _ptr(hm), OPB_HOST, planes, h, w, int(bool(mirror)),
                                                         float(thresh), _ptr(out), _ptr(valid)))
        return self._keypoint_list(out, valid)

    def image_detail(self, img):
        pk = np.empty((self.max_peaks, 5), np.float64)
        n_pk, n_sub = C.c_int(0), C.c_int(0)
        cap = 19 * 1024
        conn = np.empty((cap, 3), np.float64)
        counts = np.zeros(N_LIMBS, np.int32)
        subs = np.empty((self.max_persons, 20), np.float64)
        self._check(self.lib.opb_get_image_detail(self.ctx, img, _ptr(pk), self.max_peaks, C.byref(n_pk), _ptr(conn),
                                                  cap, _ptr(counts), _ptr(subs), self.max_persons, C.byref(n_sub)))
        conns, o = [], 0
        for c in counts:
            conns.append(conn[o:o + c].copy() if c else np.zeros((0, 3)))
            o += int(c)
        return pk[:n_pk.value].copy(), conns, subs[:n_sub.value].copy()

    # -- precise path -----------------------------------------------------------------------
    def precise_begin(self, orig_h, orig_w):
        self._check(self.lib.opb_precise_begin(self.ctx, orig_h, orig_w))

    def precise_add_scale_unpadded(self, img, stride, pad_value, scale_index, n_scales):
        """Resized but unpadded uint8 frame; pad_image (pose_detector.py:46-55) runs on the device."""
        img = np.ascontiguousarray(img, np.uint8)
        h, w, _ = img.shape
        pv = (C.c_uint8 * 3)(*[int(v) for v in pad_value])
        self._check(self.lib.opb_precise_add_scale_unpadded(self.ctx, _ptr(img), OPB_HOST, h, w, int(stride), pv,
                                                            scale_index, n_scales))

    def precise_add_scale_orig(self, orig_img, h, w, stride, pad_value, scale_index, n_scales):
        """Original uint8 frame; the cubic resize to (h, w) of pose_detector.py:443 and pad_image run on the device."""
        img = np.ascontiguousarray(orig_img, np.uint8)
        oh, ow, _ = img.shape
        pv = (C.c_uint8 * 3)(*[int(v) for v in pad_value])
        self._check(self.lib.opb_precise_add_scale_orig(self.ctx, _ptr(img), OPB_HOST, oh, ow, int(h), int(w), int(stride),
                                                        pv, scale_index, n_scales))

    def precise_add_scale(self, padded_img, pad, scale_index, n_scales):
        img = np.ascontiguousarray(padded_img, np.uint8)
        ph, pw, _ = img.shape
        self._check(self.lib.opb_precise_add_scale(self.ctx, _ptr(img), OPB_HOST, ph, pw, int(pad[0]), int(pad[1]),
                                                   scale_index, n_scales))

    def precise_finish(self, img_len):
        headers = np.empty(1, HEADER_DTYPE)
        persons = np.empty((1, self.max_persons), PERSON_DTYPE)
        self._check(self.lib.opb_precise_finish(self.ctx, float(img_len), _ptr(headers), _ptr(persons), OPB_HOST))
        return headers, persons

    def download_maps(self, h, w):
        pafs = np.empty((38, h, w), np.float32)
        heat = np.empty((19, h, w), np.float32)
        self._check(self.lib.opb_download_maps(self.ctx, _ptr(pafs), _ptr(heat), OPB_HOST))
        return pafs, heat

    # -- Haar cascade (include/opb.h: opb_cascade_*) -------------------------------------------
    def cascade_load(self, t):
        """Load a cascade.HaarCascade into this context (one cascade per context; this replaces the previous one)."""
        arrs = [np.ascontiguousarray(a, dt) for a, dt in
                ((t.stage_ntrees, np.int32), (t.stage_threshold, np.float32), (t.stump_feature, np.int32),
                 (t.stump_threshold, np.float32), (t.stump_left, np.float32), (t.stump_right, np.float32),
                 (t.rects, np.int32), (t.weights, np.float32))]
        ntrees, sthr, feat, thr, left, right, rects, weights = arrs
        self._check(self.lib.opb_cascade_load(self.ctx, int(t.window[0]), int(t.window[1]), len(ntrees), _ptr(ntrees),
                                              _ptr(sthr), len(feat), _ptr(feat), _ptr(thr), _ptr(left), _ptr(right),
                                              len(rects), _ptr(rects), _ptr(weights)))
        self.cascade_tables = t

    @staticmethod
    def _cascade_frame(img):
        img = np.asarray(img)
        if img.dtype != np.uint8 or not (img.ndim == 2 or (img.ndim == 3 and img.shape[2] in (1, 3))):
            raise ValueError("image must be uint8 [H, W] gray or [H, W, 3] BGR, got %s %s" % (img.dtype, img.shape))
        img = np.ascontiguousarray(img)
        return img, img.shape[0], img.shape[1], (1 if img.ndim == 2 else img.shape[2])

    @staticmethod
    def _cascade_args(scale_factor, min_neighbors, min_size, max_size):
        vals = [float(scale_factor), int(min_neighbors)] + [int(v) for v in tuple(min_size) + tuple(max_size)]
        if len(vals) != 6:
            raise ValueError("minSize and maxSize must be (w, h) pairs")
        if not vals[0] > 1 or min(vals[1:]) < 0:
            raise ValueError("scaleFactor must be > 1 and minNeighbors, minSize, maxSize must not be negative")
        return vals

    def cascade_detect(self, img, scale_factor, min_neighbors, min_size, max_size, cap=4096):
        """detectMultiScale on the device (opb_cascade_detect): int32 [n, 4] rects sorted by (y, x, w, h)."""
        img, h, w, ch = self._cascade_frame(img)
        sf, mn, min_w, min_h, max_w, max_h = self._cascade_args(scale_factor, min_neighbors, min_size, max_size)
        out = np.empty((cap, 4), np.int32)
        n = C.c_int(0)
        self._check(self.lib.opb_cascade_detect(self.ctx, _ptr(img), OPB_HOST, h, w, ch, sf, mn, min_w, min_h, max_w,
                                                max_h, _ptr(out), cap, C.byref(n)))
        return out[:n.value].copy()

    def face_detect_frame(self, img, scale_factor, min_neighbors, min_size, max_size, crop_scale, net_size, thresh,
                          cap=1024):
        """camera_face_demo.py's frame on the device (opb_face_detect_frame): (rects int32 [n, 4], keypoint lists,
        crop (left, top) pairs)."""
        img, h, w, ch = self._cascade_frame(img)
        if ch != 3:
            raise ValueError("face_detect_frame needs a BGR [H, W, 3] frame")
        sf, mn, min_w, min_h, max_w, max_h = self._cascade_args(scale_factor, min_neighbors, min_size, max_size)
        planes = max(getattr(self, "kp_channels", 0) - 1, 0)   # 0 on a context without FaceNet: OPB_ERR_STATE
        rects = np.empty((cap, 4), np.int32)
        out = np.empty((cap, planes, 3), np.float64)
        valid = np.empty((cap, planes), np.int32)
        left_top = np.empty((cap, 2), np.int32)
        n = C.c_int(0)
        self._check(self.lib.opb_face_detect_frame(self.ctx, _ptr(img), OPB_HOST, h, w, sf, mn, min_w, min_h, max_w,
                                                   max_h, float(crop_scale), int(net_size), float(thresh), _ptr(rects),
                                                   cap, C.byref(n), _ptr(out), _ptr(valid), _ptr(left_top)))
        k = n.value
        return (rects[:k].copy(), [self._keypoint_list(o, v) for o, v in zip(out[:k], valid[:k])],
                [(int(a), int(b)) for a, b in left_top[:k]])

    # -- the whole-body frame (include/opb.h: opb_whole_body_frame) ---------------------------------
    def whole_body_frame(self, face_engine, hand_engine, img, in_h, in_w, map_h, map_w, img_len, face_net_size,
                         face_thresh, hand_net_size, hand_thresh, draw=True, inject_paf=None, inject_heat=None):
        """demo.py's frame on the device with this (pose) context and the FaceNet / HandNet contexts: returns
        (headers[1], persons[1, max_persons], parts (WB_PART_DTYPE [n]), face keypoint lists by row, hand keypoint lists
        by row, picture [H,W,3] uint8 or None).  inject_*: device pointers (ints) or None, as in detect_batch."""
        img = np.ascontiguousarray(img, np.uint8)
        oh, ow, _ = img.shape
        headers = np.empty(1, HEADER_DTYPE)
        persons = np.empty((1, self.max_persons), PERSON_DTYPE)
        cap = 3 * self.max_persons                     # every person has at most a face and two hands
        parts = np.empty(cap, WB_PART_DTYPE)
        fpl = max(getattr(face_engine, "kp_channels", 0) - 1, 0)
        hpl = max(getattr(hand_engine, "kp_channels", 0) - 1, 0)
        face_out, face_valid = np.empty((cap, fpl, 3), np.float64), np.empty((cap, fpl), np.int32)
        hand_out, hand_valid = np.empty((cap, hpl, 3), np.float64), np.empty((cap, hpl), np.int32)
        picture = np.empty_like(img) if draw else None
        n = C.c_int(0)
        self._check(self.lib.opb_whole_body_frame(
            self.ctx, face_engine.ctx, hand_engine.ctx, _ptr(img), OPB_HOST, oh, ow, in_h, in_w, map_h, map_w,
            float(img_len), C.c_void_p(int(inject_paf)) if inject_paf else None,
            C.c_void_p(int(inject_heat)) if inject_heat else None, int(face_net_size), float(face_thresh),
            int(hand_net_size), float(hand_thresh), _ptr(headers), _ptr(persons), _ptr(parts), cap, C.byref(n),
            _ptr(face_out), _ptr(face_valid), _ptr(hand_out), _ptr(hand_valid), _ptr(picture)))
        parts = parts[:n.value].copy()
        n_face = int((parts["kind"] == PART_FACE).sum())
        faces = [self._keypoint_list(o, v) for o, v in zip(face_out[:n_face], face_valid[:n_face])]
        hands = [self._keypoint_list(o, v) for o, v in zip(hand_out[:n.value - n_face], hand_valid[:n.value - n_face])]
        return headers, persons, parts, faces, hands, picture

    def whole_body_batch(self, face_engine, hand_engine, frames, in_h, in_w, map_h, map_w, img_len, face_net_size,
                         face_thresh, hand_net_size, hand_thresh, draw=True, inject_paf=None, inject_heat=None):
        """opb_whole_body_batch on N equally sized frames [N,H,W,3] uint8: returns (headers[N], persons[N, max_persons],
        parts (WB_PART_DTYPE [k]), frame_parts int [N + 1], face keypoint lists by row, hand keypoint lists by row,
        pictures [N,H,W,3] uint8 or None).  A frame's record status raises what raise_for_status raises for it.
        inject_*: device pointers (ints) to [N,38|19,in_h/8,in_w/8] maps, or None."""
        frames = np.ascontiguousarray(frames, np.uint8)
        n, oh, ow, _ = frames.shape
        headers = np.zeros(n, HEADER_DTYPE)
        persons = np.empty((n, self.max_persons), PERSON_DTYPE)
        cap = 3 * self.max_persons * n                 # every person has at most a face and two hands
        parts = np.empty(cap, WB_PART_DTYPE)
        frame_parts = np.zeros(n + 1, np.int32)
        fpl = max(getattr(face_engine, "kp_channels", 0) - 1, 0)
        hpl = max(getattr(hand_engine, "kp_channels", 0) - 1, 0)
        face_out, face_valid = np.empty((cap, fpl, 3), np.float64), np.empty((cap, fpl), np.int32)
        hand_out, hand_valid = np.empty((cap, hpl, 3), np.float64), np.empty((cap, hpl), np.int32)
        pictures = np.empty_like(frames) if draw else None
        k = C.c_int(0)
        rc = self.lib.opb_whole_body_batch(
            self.ctx, face_engine.ctx, hand_engine.ctx, _ptr(frames), OPB_HOST, n, oh, ow, in_h, in_w, map_h, map_w,
            float(img_len), C.c_void_p(int(inject_paf)) if inject_paf else None,
            C.c_void_p(int(inject_heat)) if inject_heat else None, int(face_net_size), float(face_thresh),
            int(hand_net_size), float(hand_thresh), _ptr(headers), _ptr(persons), _ptr(parts), cap, C.byref(k),
            _ptr(frame_parts), _ptr(face_out), _ptr(face_valid), _ptr(hand_out), _ptr(hand_valid), _ptr(pictures))
        if rc != 0:
            bad = np.flatnonzero(headers["status"] != 0)
            if len(bad) and int(headers["status"][bad[0]]) == rc:   # a frame's record status, as detect_batch raises it
                self.raise_for_status(rc)
            self._check(rc)
        parts = parts[:k.value].copy()
        n_face = int((parts["kind"] == PART_FACE).sum())
        faces = [self._keypoint_list(o, v) for o, v in zip(face_out[:n_face], face_valid[:n_face])]
        hands = [self._keypoint_list(o, v) for o, v in zip(hand_out[:k.value - n_face], hand_valid[:k.value - n_face])]
        return headers, persons, parts, frame_parts, faces, hands, pictures

    def test_whole_body_boxes_batch(self, headers, persons, sx, sy):
        """Test hook: the crop-box kernel on the host records of N frames, headers (HEADER_DTYPE [N]) and persons
        (PERSON_DTYPE [N, cap]), in one launch -> per frame a dict with status, unit [cap], boxes [cap,3,4],
        present [cap], face / hand (CROP_DTYPE, the frame's compacted tables) and parts int32 [k, 3] (person, side,
        row)."""
        hd = np.ascontiguousarray(headers, HEADER_DTYPE)
        rec = np.ascontiguousarray(persons, PERSON_DTYPE)
        n, cap = rec.shape
        assert len(hd) == n
        counts = np.empty((n, 4), np.int32)
        unit = np.empty((n, cap), np.float64)
        boxes = np.empty((n, cap, 3, 4), np.int32)
        present = np.empty((n, cap), np.int32)
        face = np.empty((n, cap), CROP_DTYPE)
        hand = np.empty((n, 2 * cap), CROP_DTYPE)
        parts = np.empty((n, 3 * cap, 4), np.int32)
        self._check(self.lib.opb_test_whole_body_boxes_batch(self.ctx, _ptr(hd), _ptr(rec), n, cap, float(sx), float(sy),
                                                             _ptr(counts), _ptr(unit), _ptr(boxes), _ptr(present),
                                                             _ptr(face), _ptr(hand), _ptr(parts)))
        out = []
        for f in range(n):
            status, nf, nh, k = (int(v) for v in counts[f])
            out.append(dict(status=status, unit=unit[f], boxes=boxes[f], present=present[f], face=face[f, :nf].copy(),
                            hand=hand[f, :nh].copy(), parts=parts[f, :k][:, [1, 0, 2]].copy()))
        return out

    def test_whole_body_boxes(self, persons, sx, sy):
        """Test hook: the crop-box kernel on host person records (PERSON_DTYPE [n]) -> (unit lengths float64 [n],
        boxes int32 [n, 3, 4] (face, left, right), present bits int32 [n], kept parts int32 [k, 2] (person, side))."""
        rec = np.ascontiguousarray(persons, PERSON_DTYPE)
        n = len(rec)
        unit = np.empty(max(n, 1), np.float64)
        boxes = np.zeros((max(n, 1), 3, 4), np.int32)
        present = np.empty(max(n, 1), np.int32)
        parts = np.empty((3 * max(n, 1), 2), np.int32)
        k = C.c_int(0)
        self._check(self.lib.opb_test_whole_body_boxes(self.ctx, _ptr(rec), n, float(sx), float(sy), _ptr(unit),
                                                       _ptr(boxes), _ptr(present), _ptr(parts), C.byref(k)))
        return unit[:n], boxes[:n], present[:n], parts[:k.value].copy()

    def test_cascade_windows(self, img, scale_factor, min_size=(0, 0), max_size=(0, 0)):
        """Test hook: (codes int32 [n], stage sums float64 [n]) of every window of every scale, before the skip rule."""
        img, h, w, ch = self._cascade_frame(img)
        sf, _, min_w, min_h, max_w, max_h = self._cascade_args(scale_factor, 0, min_size, max_size)
        n = C.c_int(0)
        rc = self.lib.opb_test_cascade_windows(self.ctx, _ptr(img), OPB_HOST, h, w, ch, sf, min_w, min_h, max_w, max_h,
                                               None, None, 0, C.byref(n))
        if rc not in (0, ERR_CAPACITY):
            self._check(rc)
        codes = np.empty(max(n.value, 1), np.int32)
        sums = np.empty(max(n.value, 1), np.float64)
        self._check(self.lib.opb_test_cascade_windows(self.ctx, _ptr(img), OPB_HOST, h, w, ch, sf, min_w, min_h, max_w,
                                                      max_h, _ptr(codes), _ptr(sums), len(codes), C.byref(n)))
        return codes[:n.value], sums[:n.value]

    # -- instrumentation ----------------------------------------------------------------------
    def device_buffer(self, which):
        return self.lib.opb_device_buffer(self.ctx, which)

    def launch_count(self):
        return int(self.lib.opb_launch_count(self.ctx))

    def time_stage(self, stage, reps=10):
        ms = C.c_float(0)
        self._check(self.lib.opb_time_stage(self.ctx, stage.encode(), reps, C.byref(ms)))
        return float(ms.value)

    def test_conv(self, x, W, b, relu, precision, pool=False):
        x = np.ascontiguousarray(x, np.float32)
        W = np.ascontiguousarray(W, np.float32)
        b = np.ascontiguousarray(b, np.float32)
        n, h, w, cin = x.shape
        cout, _, ks, _ = W.shape
        y = np.empty((n, h // 2, w // 2, cout) if pool else (n, h, w, cout), np.float32)
        self._check(self.lib.opb_test_conv(self.ctx, _ptr(x), n, h, w, cin, _ptr(W), _ptr(b), cout, ks,
                                           int(bool(relu)) | (2 if pool else 0), int(precision), _ptr(y)))
        return y

    def test_conv_first(self, x, W, b, precision, u8_denom=255.0):
        """conv1_1 alone: x uint8 [N,H,W,3] BGR or float32 [N,3,H,W] (preprocessed), W [64,3,3,3], b [64].
        Returns the raw output tensor as uint8 [N,H,W,128] (fast) or [N,H,W,256] (parity, compensated)."""
        is_u8 = np.asarray(x).dtype == np.uint8
        x = np.ascontiguousarray(x, np.uint8 if is_u8 else np.float32)
        W = np.ascontiguousarray(W, np.float32)
        b = np.ascontiguousarray(b, np.float32)
        if is_u8:
            n, h, w, _ = x.shape
        else:
            n, _, h, w = x.shape
        out = np.empty((n, h, w, 128 if int(precision) == PRECISION_FAST else 256), np.uint8)
        self._check(self.lib.opb_test_conv_first(self.ctx, _ptr(x), int(is_u8), n, h, w, float(u8_denom), _ptr(W),
                                                 _ptr(b), int(precision), _ptr(out)))
        return out

    def test_chain_convs(self, n, h, w):
        """The conv launches of the loaded model's chain at (n, h, w): a CONV_RECORD_DTYPE array in launch order."""
        count = C.c_int(0)
        rc = self.lib.opb_test_chain_convs(self.ctx, int(n), int(h), int(w), None, 0, C.byref(count))
        if rc not in (0, ERR_CAPACITY):
            self._check(rc)
        recs = np.zeros(count.value, CONV_RECORD_DTYPE)
        self._check(self.lib.opb_test_chain_convs(self.ctx, int(n), int(h), int(w), _ptr(recs), len(recs), C.byref(count)))
        return recs

    def test_chain_conv_run(self, n, h, w, index, in0, in1, out_io, out32=(None, None)):
        """Runs conv launch `index` of that chain alone.  in0 / in1: raw input tensors (uint8 arrays of the whole
        tensor; in1 only when problem 1 reads another tensor); out_io (uint8, whole output tensor) and the float32 maps
        of out32 are uploaded as prior content and overwritten in place with what the launch left there."""
        arrs = [in0, in1, out_io] + list(out32)
        for a in arrs:
            assert a is None or (isinstance(a, np.ndarray) and a.flags.c_contiguous)
        self._check(self.lib.opb_test_chain_conv_run(self.ctx, int(n), int(h), int(w), int(index), *map(_ptr, arrs)))

    def test_keypoint_stages(self, frames, crops, net_size, planes, maps, thresh, tail=4096):
        """Test hook: the face / hand crop pass (opb_test_keypoint_stages) on frames uint8 [F,H,W,3], crop rows
        (KP_STAGE_CROP_DTYPE, or (left, top, right, bottom, flip, frame, vh, vw) tuples) and injected maps float32
        [n][planes + 1][net/8][net/8].  Every output holds `tail` elements past its size.  Returns a dict: sizes
        (canvas bytes, map floats, records), canvas uint8, up / tmp / smooth float32, records (CHANNEL_MAX_DTYPE),
        out float64 [n, planes, 3], valid int32 [n, planes] and keypoints (one keypoint list per crop)."""
        fr = np.ascontiguousarray(frames, np.uint8)
        rows = np.ascontiguousarray(np.array([tuple(r) for r in crops], KP_STAGE_CROP_DTYPE))
        mp = np.ascontiguousarray(maps, np.float32)
        n_frames, fh, fw, _ = fr.shape
        n = len(rows)
        sizes = np.zeros(3, np.int64)

        def call(canvas, cc, up, tmp, smooth, mc, rec, rc_, out, valid):
            return self.lib.opb_test_keypoint_stages(self.ctx, _ptr(fr), n_frames, fh, fw, _ptr(rows), n, int(net_size),
                                                     int(planes), _ptr(mp), float(thresh), _ptr(canvas), cc, _ptr(up),
                                                     _ptr(tmp), _ptr(smooth), mc, _ptr(rec), rc_, _ptr(out),
                                                     _ptr(valid), _ptr(sizes))
        rc = call(None, 0, None, None, None, 0, None, 0, None, None)
        if rc != ERR_CAPACITY:
            self._check(rc)
        cb, nf, nr = (int(v) + tail for v in sizes)
        canvas = np.empty(cb, np.uint8)
        up, tmp, smooth = (np.empty(nf, np.float32) for _ in range(3))
        records = np.empty(nr, CHANNEL_MAX_DTYPE)
        out = np.empty((n, planes, 3), np.float64)
        valid = np.empty((n, planes), np.int32)
        self._check(call(canvas, cb, up, tmp, smooth, nf, records, nr, out, valid))
        return dict(sizes=tuple(int(v) for v in sizes), canvas=canvas, up=up, tmp=tmp, smooth=smooth, records=records,
                    out=out, valid=valid, keypoints=[self._keypoint_list(o, v) for o, v in zip(out, valid)])
