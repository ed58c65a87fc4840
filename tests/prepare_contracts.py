"""The contracts of dh_prepare_frames_u8 and dh_pose_to_image_f32 in float64 / integers, and their stand-ins on the
stand-in device -- TEST INFRASTRUCTURE (never imported by the product).

`install()` registers the two stand-ins with tests/fake_cuda.py (and keeps dh_prepare_frames_workspace, a host-only
entry point, real) before installing the stand-in device with arithmetic, so that FramePipeline.from_device runs on the
CPU through the product's own record packing and argument marshalling."""
import ctypes as C

import numpy as np

FRAME_EMPTY, FRAME_TOO_LARGE, FRAME_BAD_BOX = 1, 2, 4


def frame_box(objpos, winsize, max_crop, image_ok=True):
    """dh_prepare_frames_u8's box of one record -> (box [x0, y0, x1, y1] or None, status bits): the edges cx -+ ww / 2,
    cy -+ wh / 2 truncated toward zero; not finite or outside int32 (or a bad image record) is FRAME_BAD_BOX, a window
    under one pixel FRAME_EMPTY, one over max_crop = (w, h) FRAME_TOO_LARGE"""
    (cx, cy), (ww, wh) = [float(v) for v in objpos], [float(v) for v in winsize]
    edges = [cx - ww / 2, cy - wh / 2, cx + ww / 2, cy + wh / 2]
    if not image_ok or not np.all(np.isfinite([cx, cy, ww, wh])) or \
            not all(-2147483649.0 < e < 2147483648.0 for e in edges):
        return None, FRAME_BAD_BOX
    box = [int(e) for e in edges]
    cw, ch = box[2] - box[0], box[3] - box[1]
    if cw < 1 or ch < 1:
        return None, FRAME_EMPTY
    if cw > max_crop[0] or ch > max_crop[1]:
        return None, FRAME_TOO_LARGE
    return box, 0


def prepare_frame(img, box, out_wh, hflip, channel_power=1):
    """a usable frame of dh_prepare_frames_u8 -> (frame (out_h, out_w, 3) float32, afmat (3, 3)): the crop -> Pillow
    resize -> [flip] -> normalize_channels of the oracle, and translate -> scale -> [flip] -> normalise as matrices"""
    from oracle import preprocess as OP
    rw, rh = out_wh

    def m(*rows):
        return np.array(rows, np.float64)
    cw, ch = box[2] - box[0], box[3] - box[1]
    a = np.dot(m([rw / cw, 0, 0], [0, rh / ch, 0], [0, 0, 1]), m([1, 0, -box[0]], [0, 1, -box[1]], [0, 0, 1]))
    if hflip:
        a = np.dot(m([1, 0, rw], [0, 1, 0], [0, 0, 1]), np.dot(m([-1, 0, 0], [0, 1, 0], [0, 0, 1]), a))
    a = np.dot(m([1 / rw, 0, 0], [0, 1 / rh, 0], [0, 0, 1]), a)
    return OP.eval_frame(img, tuple(box), (rw, rh), hflip=bool(hflip), channel_power=channel_power), a


def pose_to_image(poses, afmat):
    """dh_pose_to_image_f32: poses (n, points, >= 2), already widened to float64, through inv(afmat) ((n | 1, 3, 3); a
    singular map gives NaN) -> (n, points, 2)"""
    M = np.stack([np.linalg.inv(a) if np.linalg.matrix_rank(a) == 3 else np.full((3, 3), np.nan) for a in afmat])
    M = np.broadcast_to(M, (len(poses), 3, 3))
    return np.einsum('nij,nkj->nki', M[:, :2, :2], poses[:, :, :2]) + M[:, None, :2, 2]


# ---- stand-ins: the contracts above from the entry points' raw ctypes arguments -----------------------------------------

def _prepare_frames(ctx, boxes, n, mw, mh, rh, rw, power, ws, ws_bytes, out, afmat, status, stream):
    """csrc/preprocess.cu dh_prepare_frames_u8: per box record the box, its status and, when usable, the frame and the
    afmat; a flagged frame is NaN in its elements and its afmat"""
    import fake_cuda as F
    from deephar_b200._ffi import dh_frame_box
    recs = C.cast(boxes, C.POINTER(dh_frame_box))
    o, A = F._dense(out, n, rh, rw, 3), F._dense64(afmat, n, 3, 3)
    st = np.ctypeslib.as_array(C.cast(status, C.POINTER(C.c_int32)), shape=(n,))
    pw = 1 if not power else tuple(float(v) for v in F._f32(power, 3))
    for i in range(n):
        r = recs[i]
        h, w, stride = int(r.h), int(r.w), int(r.stride)
        image_ok = h >= 0 and w >= 0 and stride >= 3 * w and bool(r.data or not h * w)
        box, st[i] = frame_box(r.objpos, r.winsize, (mw, mh), image_ok)
        if box is None:
            o[i], A[i] = np.nan, np.nan
            continue
        img = np.ctypeslib.as_array(C.cast(r.data, C.POINTER(C.c_uint8)), shape=(h, stride))[:, :w * 3].reshape(h, w, 3)
        o[i], A[i] = prepare_frame(img, box, (rw, rh), int(r.hflip) == 1, pw)


def _pose_to_image(ctx, poses, afmat, per_sample, out, stream):
    """csrc/postprocess.cu dh_pose_to_image_f32: the view's (x, y) widened to float64, through inv(afmat)"""
    import fake_cuda as F
    v = poses.contents
    n, pts = int(v.n), int(v.h) * int(v.w)
    P = F._in(poses).reshape(n, pts, int(v.c))
    F._dense64(out, n, pts, 2)[...] = pose_to_image(P, F._dense64(afmat, n if per_sample else 1, 3, 3))


def install():
    """the stand-in device with arithmetic, these two entry points included"""
    import fake_cuda as F
    F.ARITHMETIC['dh_prepare_frames_u8'] = _prepare_frames
    F.ARITHMETIC['dh_pose_to_image_f32'] = _pose_to_image
    F.HOST_ENTRY_POINTS = F.HOST_ENTRY_POINTS + ('dh_prepare_frames_workspace',)
    return F.install(arithmetic=True)
