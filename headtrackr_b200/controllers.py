"""Host mirror of the reference's head-coupled camera controller, headtrackr.controllers.three.
realisticAbsoluteCameraControl (src/controllers.js:28-68), over a minimal perspective camera.

The listener body runs in fp64 in JavaScript's evaluation order (Python floats are IEEE doubles, and Python does not
fuse a*b+c), so every field is bit-identical to the reference's.  `updateProjectionMatrix` is three.js r48's as
DESIGN.md 5.4 (f10) restates it: the projection and view matrices in fp64, rounded once to float32, as (4, 4) numpy
arrays indexed [row, col] (the library stores them column-major, the WebGL layout).

The device runs the same controller per stream during the tick (Context.tracker_set_camera, the "camera" key of
streams.TrackerSet).  Pinned against the reference's own controllers.js executed by oracle/jsmini.py
(tests/golden/reference_js_controllers.json, tools/make_goldens_controllers.py, tests/test_controllers_host.py).
"""
import math

import numpy as np


def _div(a, b):
    """JavaScript's a / b (IEEE: x / 0 is +-Infinity or NaN)"""
    if b == 0.0:
        if a != a or a == 0.0:
            return math.nan
        return -math.inf if (a < 0) != (math.copysign(1.0, b) < 0) else math.inf
    return a / b


def look_at(eye, target):
    """R of r48's lookAt(eye -> target, up = +y) without its epsilon nudge: columns x, y, z as a (3, 3) fp64 array;
    ValueError for a degenerate lookAt (eye == target, a view direction parallel to up)"""
    z = [float(eye[i]) - float(target[i]) for i in range(3)]
    zn = math.sqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2])
    if not 0.0 < zn < math.inf:
        raise ValueError("degenerate lookAt: the camera is at its target")
    z = [v / zn for v in z]
    x = [z[2], 0.0, -z[0]]
    xn = math.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2])
    if not xn > 0.0:
        raise ValueError("degenerate lookAt: the view direction is parallel to up")
    x = [v / xn for v in x]
    y = [z[1] * x[2] - z[2] * x[1], z[2] * x[0] - z[0] * x[2], z[0] * x[1] - z[1] * x[0]]
    r = np.array([x, y, z], np.float64).T
    if not (np.abs(r) <= 1.0).all():
        raise ValueError("degenerate lookAt")
    return r


def frustum(l, r, b, t, n, f):
    """r48 makeFrustum -> float32 (4, 4)"""
    m = np.zeros((4, 4), np.float64)
    m[0, 0] = _div(2 * n, r - l)
    m[1, 1] = _div(2 * n, t - b)
    m[0, 2] = _div(r + l, r - l)
    m[1, 2] = _div(t + b, t - b)
    m[2, 2] = _div(-(f + n), f - n)
    m[3, 2] = -1.0
    m[2, 3] = _div(-2 * f * n, f - n)
    return m.astype(np.float32)


def projection_matrix(fov, aspect, near, far, view=None):
    """r48 updateProjectionMatrix: with a view offset (fullWidth, fullHeight, x, y, width, height) the off-axis
    frustum, else makePerspective(fov, aspect, near, far)"""
    if view is not None:
        fw, fh, x, y, w, h = view
        a = _div(fw, fh)
        top = math.tan(fov * math.pi / 360) * near
        left = -(a * top)
        width, height = 2 * (a * top), 2 * top
        return frustum(left + _div(x * width, fw), left + _div((x + w) * width, fw),
                       top - _div((y + h) * height, fh), top - _div(y * height, fh), near, far)
    ymax = near * math.tan(fov * math.pi / 360)
    return frustum(-ymax * aspect, ymax * aspect, -ymax, ymax, near, far)


def view_matrix(rot, position):
    """inverse(T(position) R) = R^T T(-position) -> float32 (4, 4)"""
    m = np.zeros((4, 4), np.float64)
    for r in range(3):
        a = [float(v) for v in rot[:, r]]
        m[r, :3] = a
        m[r, 3] = -(a[0] * position[0] + a[1] * position[1] + a[2] * position[2])
    m[3, 3] = 1.0
    return m.astype(np.float32)


class PerspectiveCamera:
    """The part of three.js r48's PerspectiveCamera that realisticAbsoluteCameraControl uses"""

    def __init__(self, fov=50.0, aspect=1.0, near=0.1, far=2000.0):
        self.fov, self.aspect, self.near, self.far = float(fov), float(aspect), float(near), float(far)
        self.position = [0.0, 0.0, 0.0]
        self.view = None                        # setViewOffset's arguments
        self.rotation = np.eye(3)
        self.projectionMatrix = None
        self.matrixWorldInverse = None
        self.updateProjectionMatrix()

    def lookAt(self, target):
        self.rotation = look_at(self.position, target)
        self.matrixWorldInverse = view_matrix(self.rotation, self.position)

    def setViewOffset(self, fullWidth, fullHeight, x, y, width, height):
        self.view = [fullWidth, fullHeight, x, y, width, height]
        self.updateProjectionMatrix()

    def updateProjectionMatrix(self):
        self.projectionMatrix = projection_matrix(self.fov, self.aspect, self.near, self.far, self.view)
        self.matrixWorldInverse = view_matrix(self.rotation, self.position)


class realisticAbsoluteCameraControl:
    """src/controllers.js:28-68: constructs the camera (position = fixedPosition, lookAt(lookAt)) and moves it on
    every headtrackingEvent passed to handleEvent.  tracker: a main.Tracker (addEventListener(type, fn)) or a
    streams.TrackerSet (with `stream`, the index whose events it hears); None: call handleEvent yourself.
    `events` counts the headtrackingEvents applied."""

    def __init__(self, camera, scaling, fixedPosition, lookAt, params=None, tracker=None, stream=None):
        params = {} if params is None else params
        self.screenHeight = float(params.get("screenHeight", 20.0))
        self.damping = float(params.get("damping", 1.0))
        self.camera, self.scaling = camera, float(scaling)
        self.fixedPosition = [float(v) for v in fixedPosition]
        camera.position = list(self.fixedPosition)
        camera.lookAt([float(v) for v in lookAt])
        self.wh = self.screenHeight * self.scaling
        self.ww = self.wh * camera.aspect
        self.events = 0
        if tracker is not None:
            if stream is None:
                tracker.addEventListener("headtrackingEvent", self.handleEvent)
            else:
                tracker.addEventListener(lambda k, e: self.handleEvent(e) if k == stream and
                                         e.get("type") == "headtrackingEvent" else None)

    def handleEvent(self, event):
        """the listener of src/controllers.js:48-67"""
        x, y, z = float(event["x"]), float(event["y"]), float(event["z"])
        s, d, cam = self.scaling, self.damping, self.camera
        xOffset = 0.0 if x > 0 else -x * 2 * d * s
        yOffset = 0.0 if y < 0 else y * 2 * d * s
        cam.view = [self.ww + abs(x * 2 * d * s), self.wh + abs(y * d * 2 * s), xOffset, yOffset, self.ww, self.wh]
        cam.position = [self.fixedPosition[0] + (x * s * d), self.fixedPosition[1] + (y * s * d),
                        self.fixedPosition[2] + (z * s)]
        cam.fov = _div(math.atan(_div(self.wh / 2 + abs(y * s * d), abs(z * s))) * 360, math.pi)
        self.events += 1
        cam.updateProjectionMatrix()

    def state(self):
        """the camera as an ht_camera decodes (Context.camera_from_bytes)"""
        c = self.camera
        return dict(position=list(c.position), fov=c.fov, view=list(c.view) if c.view else [0.0] * 6,
                    events=self.events, has_view_offset=int(c.view is not None), projection=c.projectionMatrix,
                    view_matrix=c.matrixWorldInverse)
