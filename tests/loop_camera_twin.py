"""The cv2 / numpy twin of findConnection (oracle/loop_verify.py) for MEI and KANNALA_BRANDT cameras (test infrastructure).

computeBRIEFPoint lifts each FAST corner with the key frame's camera, m_camera->liftProjective, and divides by z
(pose_graph/src/keyframe.cpp:108); m_camera is read from the tracker's YAML file.  Everything else in findConnection is
camera-independent, so the key frame here is the PINHOLE twin's with its corners lifted through oracle/camera_models.py and
stored as float, like the reference's cv::Point2f."""
import numpy as np

from oracle import camera_models as cm
from oracle import loop_verify as olv


def lift_corners(camera_model, intr, xi, px):
    """liftProjective / z of the pixels px (n, 2) for camera_model 0 PINHOLE, 1 MEI, 2 KANNALA_BRANDT, intrinsics in the
    tracker's order for that model (MEI gamma1 gamma2 u0 v0 k1 k2 p1 p2; KANNALA_BRANDT mu mv u0 v0 k2 k3 k4 k5)."""
    if camera_model == 0:
        return olv.lift_pinhole(intr, px)
    a, b, c, d, e, f, g, h = [float(v) for v in intr]
    px = np.asarray(px, np.float64).reshape(-1, 2)
    if camera_model == 1:
        rays = [cm.mei_lift(u, v, float(xi), e, f, g, h, a, b, c, d) for u, v in px]
    else:
        rays = [cm.kb_lift(u, v, e, f, g, h, a, b, c, d) for u, v in px]
    rays = np.array(rays).reshape(-1, 3)
    return rays[:, :2] / rays[:, 2:3]


class KeyFrame(olv.KeyFrame):
    """olv.KeyFrame whose corners are lifted with the given camera (intr in that model's order)."""

    def __init__(self, image, vio_T, vio_R, p3d, uv, norm, ids, pattern, intr, camera_model=0, xi=0.0):
        super().__init__(image, vio_T, vio_R, p3d, uv, norm, ids, pattern, intr)
        if camera_model != 0:
            self.kp_norm = lift_corners(camera_model, intr, xi, self.kp.astype(np.float64)).astype(np.float32)
