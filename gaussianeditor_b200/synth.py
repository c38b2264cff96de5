"""Seeded synthetic Gaussian clouds and cameras for the BASELINE.json configs.

There is no dataset in the build container (and no network), so every workload
is generated from a fixed seed with numpy and is therefore bit-identical on the
build box and the GPU box.  The generators follow SURVEY.md section 8(d):

  cfg 1  10k   uniform cube        SH deg 0   256x256    (oracle plumbing)
  cfg 2  100k  uniform cube        SH deg 0   800x800
  cfg 3  1M    "bicycle-shaped"    SH deg 3   1600x1200  (headline)
  cfg 4  5M    "bicycle-shaped"    SH deg 3   1920x1080
  cfg 5  500k  "bicycle" x0.5      SH deg 3   512x512    (edit loop stand-in)

Camera conventions mirror the reference's ``Simple_Camera``
(/root/reference/gaussiansplatting/scene/cameras.py:86-94 and
utils/graphics_utils.py:38-88): ``viewmatrix`` is the TRANSPOSED world-to-camera
matrix, ``projmatrix`` = viewmatrix @ P^T (also transposed), znear 0.01,
zfar 100, camera looks down +z.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

SH_C0 = 0.28209479177387814

# Calibration (SURVEY.md 8(d): "calibrate, log, don't tune silently"): with the survey's nominal
# base scale 0.012 the cfg-3 cloud gives R/V = 21.3 and R/Ntile = 1732 on camera 0 -- outside the
# target band R/V 6-12, R/Ntile 800-1600 of real Mip-NeRF360 scenes.  0.65 x 0.012 gives
# R/V = 10.9, R/Ntile = 880 (measured with the CPU oracle), so that is what every config uses.
BICYCLE_BASE_SCALE = 0.012 * 0.65


@dataclass
class Cloud:
    """Activated Gaussian parameters, exactly what GaussianRasterizer.forward takes."""
    means3D: np.ndarray    # [P,3] f32
    scales: np.ndarray     # [P,3] f32 (already exp-ed)
    rotations: np.ndarray  # [P,4] f32 (already normalised, r,x,y,z)
    opacities: np.ndarray  # [P,1] f32 (already sigmoid-ed)
    shs: np.ndarray        # [P,M,3] f32
    sh_degree: int


@dataclass
class Camera:
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    viewmatrix: np.ndarray  # [4,4] f32, transposed W2C
    projmatrix: np.ndarray  # [4,4] f32, transposed full projection
    campos: np.ndarray      # [3] f32


def _projection(znear: float, zfar: float, tanx: float, tany: float) -> np.ndarray:
    # utils/graphics_utils.py:66-88 (getProjectionMatrix), float32 like the reference.
    top = tany * znear
    right = tanx * znear
    P = np.zeros((4, 4), dtype=np.float32)
    P[0, 0] = 2.0 * znear / (2.0 * right)
    P[1, 1] = 2.0 * znear / (2.0 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def look_at_camera(eye, target, up, width: int, height: int, *, fovx_deg: float | None = None,
                   fovy_deg: float | None = None) -> Camera:
    """Camera at ``eye`` looking at ``target``; exactly one of fovx/fovy is given, the
    other follows from the aspect ratio with square pixels."""
    eye = np.asarray(eye, dtype=np.float64)
    target = np.asarray(target, dtype=np.float64)
    up = np.asarray(up, dtype=np.float64)
    fwd = target - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(up, fwd)
    right /= np.linalg.norm(right)
    true_up = np.cross(fwd, right)
    # world -> camera rotation rows (camera x = right, y = down-ish (true_up), z = forward)
    Rw2c = np.stack([right, true_up, fwd], axis=0)
    W2C = np.eye(4, dtype=np.float64)
    W2C[:3, :3] = Rw2c
    W2C[:3, 3] = -Rw2c @ eye
    if fovx_deg is not None:
        tanx = math.tan(math.radians(fovx_deg) * 0.5)
        tany = tanx * height / width
    else:
        tany = math.tan(math.radians(fovy_deg) * 0.5)
        tanx = tany * width / height
    P = _projection(0.01, 100.0, tanx, tany)
    view_t = np.ascontiguousarray(W2C.astype(np.float32).T)
    proj_t = np.ascontiguousarray((view_t @ P.T).astype(np.float32))
    return Camera(height, width, float(tanx), float(tany), view_t, proj_t,
                  eye.astype(np.float32))


def ring_cameras(n: int, radius: float, elevation_deg: float, width: int, height: int,
                 fovx_deg: float) -> list[Camera]:
    cams = []
    el = math.radians(elevation_deg)
    for k in range(n):
        az = 2.0 * math.pi * k / n
        eye = (radius * math.cos(el) * math.cos(az), -radius * math.sin(el),
               radius * math.cos(el) * math.sin(az))
        cams.append(look_at_camera(eye, (0, 0, 0), (0, -1, 0), width, height, fovx_deg=fovx_deg))
    return cams


def _random_quats(rng, n):
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q.astype(np.float32)


def cube_cloud(P: int, seed: int, log_scale_mean: float, sh_degree: int = 0) -> Cloud:
    """cfg 1/2: xyz ~ U[-1,1]^3, log-scale ~ N(log s0, 0.4^2), opacity = sigmoid(N(0,2^2))."""
    rng = np.random.default_rng(seed)
    M = (sh_degree + 1) ** 2
    xyz = rng.uniform(-1.0, 1.0, (P, 3)).astype(np.float32)
    scales = np.exp(rng.normal(math.log(log_scale_mean), 0.4, (P, 3))).astype(np.float32)
    rot = _random_quats(rng, P)
    opac = (1.0 / (1.0 + np.exp(-rng.normal(0.0, 2.0, (P, 1))))).astype(np.float32)
    shs = np.zeros((P, M, 3), dtype=np.float32)
    shs[:, 0, :] = rng.standard_normal((P, 3)).astype(np.float32)
    if M > 1:
        shs[:, 1:, :] = (rng.standard_normal((P, M - 1, 3)) * 0.1).astype(np.float32)
    return Cloud(xyz, scales, rot, opac, shs, sh_degree)


def bicycle_cloud(P: int, seed: int, sh_degree: int = 3, size: float = 1.0) -> Cloud:
    """cfg 3/4/5: dense core + annulus + far shell mixture (SURVEY.md 8(d))."""
    rng = np.random.default_rng(seed)
    M = (sh_degree + 1) ** 2
    n_core = int(0.55 * P)
    n_ann = int(0.30 * P)
    n_shell = P - n_core - n_ann
    core = rng.standard_normal((n_core, 3)) * np.sqrt(np.array([1.5, 0.4, 1.5]))
    r_a = rng.uniform(3.0, 10.0, n_ann)
    th = rng.uniform(0.0, 2.0 * math.pi, n_ann)
    ann = np.stack([r_a * np.cos(th), rng.standard_normal(n_ann), r_a * np.sin(th)], axis=1)
    r_s = rng.uniform(10.0, 40.0, n_shell)
    d = rng.standard_normal((n_shell, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d[:, 1] = -np.abs(d[:, 1])  # upper hemisphere (camera "up" is -y)
    shell = d * r_s[:, None]
    xyz = np.concatenate([core, ann, shell], axis=0) * size
    r = np.linalg.norm(xyz, axis=1) / size
    base = rng.normal(np.log(BICYCLE_BASE_SCALE * np.maximum(1.0, r / 3.0)), 0.7)
    logs = base[:, None] + rng.normal(0.0, 0.5, (P, 3))
    scales = (np.exp(logs) * size).astype(np.float32)
    rot = _random_quats(rng, P)
    pick = rng.uniform(size=P) < 0.6
    logit = np.where(pick, rng.normal(2.0, 1.5, P), rng.normal(-2.0, 1.0, P))
    opac = (1.0 / (1.0 + np.exp(-logit))).astype(np.float32)[:, None]
    shs = np.zeros((P, M, 3), dtype=np.float32)
    shs[:, 0, :] = ((rng.uniform(size=(P, 3)) - 0.5) / SH_C0).astype(np.float32)
    k = 1
    for ell in range(1, sh_degree + 1):
        n = 2 * ell + 1
        shs[:, k:k + n, :] = (rng.standard_normal((P, n, 3)) * (0.15 / (1 + ell))).astype(np.float32)
        k += n
    perm = rng.permutation(P)  # interleave the three populations like a trained scene
    return Cloud(xyz.astype(np.float32)[perm], scales[perm], rot[perm], opac[perm], shs[perm],
                 sh_degree)


# ---- adversarial scenes ------------------------------------------------------------------------------------------
# Inputs where rasterizer kernels go wrong and the bicycle / cube clouds never go: needle splats, Gaussians at the
# frustum's edges, opacities at the alpha thresholds. Seeded, numpy only (same bits on every host).

def _quat_mul(a, b):
    w1, x1, y1, z1 = a.T
    w2, x2, y2, z2 = b.T
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], axis=1)


def _axis_quats(axis, angle):
    axis = np.asarray(axis, np.float64)
    q = np.zeros((angle.size, 4))
    q[:, 0] = np.cos(angle / 2)
    q[:, 1:] = np.sin(angle / 2)[:, None] * axis[None, :]
    return q


def _sh_dc(rng, P, sh_degree):
    shs = np.zeros((P, (sh_degree + 1) ** 2, 3), np.float32)
    shs[:, 0, :] = ((rng.uniform(size=(P, 3)) - 0.5) / SH_C0).astype(np.float32)
    if sh_degree > 0:
        shs[:, 1:, :] = (rng.standard_normal((P, shs.shape[1] - 1, 3)) * 0.05).astype(np.float32)
    return shs


def needle_cloud(P: int = 1000, seed: int = 0):
    """Needle splats over an empty background at 1600x1200 -> (Cloud, Camera). Axis ratio log-uniform in 10^2..10^4,
    the long axis in the image plane (tilted by at most 5 degrees) at a random angle, projected long-axis sigma
    log-uniform in 30..300 px; a third of the opacities within 5 % above 1/255, the rest uniform up to 1. Far from
    their centres the terms of the reference's `power` are ~1e5 and cancel, the regime of the render kernels'
    sub-block culling margin. SH degree 0 (tests usually pass precomputed colours)."""
    rng = np.random.default_rng(seed)
    W, H = 1600, 1200
    cam = look_at_camera((0, 0, -5), (0, 0, 0), (0, -1, 0), W, H, fovy_deg=50.0)
    focal = H / (2.0 * cam.tanfovy)
    low = rng.uniform(size=P) < 1.0 / 3.0
    opac = np.where(low, (1.0 + 0.05 * rng.uniform(size=P)) / 255.0, rng.uniform(1.0 / 255.0, 1.0, P))
    depth = 5.0 + rng.uniform(-0.5, 0.5, P)
    # projected long-axis sigma in px and image-plane angle: half of the needles spread over 30..300 px and all angles,
    # half at 280..300 px within 15 degrees of a diagonal (the largest terms, the most cancellation)
    wide = np.arange(P) % 2 == 0
    sigma = np.where(wide, np.exp(rng.uniform(np.log(30.0), np.log(300.0), P)), rng.uniform(280.0, 300.0, P))
    phi = np.where(wide, rng.uniform(0.0, np.pi, P),
                   np.pi / 4 + np.pi / 2 * rng.integers(0, 2, P) + np.radians(rng.uniform(-15.0, 15.0, P)))
    s_long = sigma * depth / focal
    ratio = np.exp(rng.uniform(np.log(1e2), np.log(1e4), (P, 2)))
    scales = np.stack([s_long, s_long / ratio[:, 0], s_long / ratio[:, 1]], axis=1)
    tilt = np.radians(rng.uniform(-5.0, 5.0, P))
    q = _quat_mul(_axis_quats((0, 0, 1), phi), _axis_quats((0, 1, 0), tilt))
    # the long axis (rotated local x) is (cos t cos phi, cos t sin phi, -sin t). The centre is placed so that the point
    # of that axis at the end of the alpha = 1/255 contour (or at 2.95 sigma, inside the 3-sigma tile square) lies in
    # the frame: that is where the terms of `power` are largest.
    axis = np.stack([np.cos(tilt) * np.cos(phi), np.cos(tilt) * np.sin(phi), -np.sin(tilt)], axis=1)
    reach = np.minimum(2.95, np.sqrt(2.0 * np.log(255.0 * opac)) * rng.uniform(0.9, 1.02, P))
    target = np.stack([rng.uniform(-0.95, 0.95, P) * cam.tanfovx * depth,
                       rng.uniform(-0.95, 0.95, P) * cam.tanfovy * depth, depth - 5.0], axis=1)
    sgn = np.where(rng.uniform(size=P) < 0.5, -1.0, 1.0)
    xyz = target - (sgn * reach * s_long)[:, None] * axis
    cloud = Cloud(xyz.astype(np.float32), scales.astype(np.float32), q.astype(np.float32),
                  opac.astype(np.float32)[:, None], _sh_dc(rng, P, 0), 0)
    return cloud, cam


def frustum_edge_cloud(seed: int = 0, sh_degree: int = 3):
    """Gaussians at the edges of the view frustum, camera at the origin looking down +z (view depth = world z exactly),
    640x480 -> (Cloud, Camera). Groups: view depths at fp32(0.2) (the near cut, `p_view.z <= 0.2`) and +-1..4 ulp and
    +-1 %; centres around |x/z| = 1.3 tan(fov) (the Jacobian clamp); centres beyond |ndc| = 1.15 whose 3-sigma radius
    still reaches the frame (read without the bulk copy of the SH row); splats larger than the frame; and scale
    vectors with one, two or three zero axes."""
    rng = np.random.default_rng(seed)
    W, H = 640, 480
    cam = look_at_camera((0, 0, 0), (0, 0, 1), (0, -1, 0), W, H, fovx_deg=61.0)  # view (x, y, z) = world (-x, -y, z)
    tx, ty = cam.tanfovx, cam.tanfovy
    z02 = np.float32(0.2)

    def ulps(k):  # fp32(0.2) moved by k ulp
        z = z02
        for _ in range(abs(k)):
            z = np.nextafter(z, np.float32(1 if k > 0 else 0))
        return np.float32(z)
    near_z = [ulps(k) for k in (-4, -1, 0, 1, 4)]
    groups = []
    # near cut: every depth 24 times, centres inside the frame, sizes a few to a few hundred pixels
    zs = np.repeat(np.array(near_z + [z02 * np.float32(0.99), z02 * np.float32(1.01)], np.float32), 24)
    n = zs.size
    xy = rng.uniform(-0.8, 0.8, (n, 2)) * np.array([tx, ty]) * zs[:, None]
    groups.append((np.concatenate([xy, zs[:, None]], 1), np.exp(rng.uniform(np.log(2e-4), np.log(5e-3), (n, 3)))))
    # Jacobian clamp: |x/z| or |y/z| within 5 % of 1.3 tan(fov)
    n = 96
    z = rng.uniform(1.5, 6.0, n)
    sgn = np.where(rng.uniform(size=(n, 2)) < 0.5, -1.0, 1.0)
    lim = 1.3 * np.array([tx, ty]) * rng.uniform(0.95, 1.05, (n, 2))
    inner = rng.uniform(-0.9, 0.9, (n, 2)) * np.array([tx, ty])
    which = rng.integers(0, 3, n)                 # clamp x, y or both
    r = np.where(np.stack([which != 1, which != 0], 1), sgn * lim, inner)
    groups.append((np.concatenate([r * z[:, None], z[:, None]], 1), np.exp(rng.uniform(np.log(0.02), np.log(0.4), (n, 3)))))
    # off-screen centres (|ndc| > 1.15) whose radius reaches into the frame
    n = 64
    z = rng.uniform(2.0, 5.0, n)
    r = rng.uniform(1.2, 2.0, (n, 2)) * np.array([tx, ty]) * sgn[:n]
    r[: n // 2, 1] = rng.uniform(-0.5, 0.5, n // 2) * ty   # half of them off-screen in x only
    groups.append((np.concatenate([r * z[:, None], z[:, None]], 1), (0.4 * z)[:, None] * rng.uniform(0.5, 1.5, (n, 3))))
    # larger than the frame
    n = 8
    z = rng.uniform(1.0, 4.0, n)
    groups.append((np.concatenate([rng.uniform(-0.3, 0.3, (n, 2)) * z[:, None], z[:, None]], 1),
                   (1.5 * z)[:, None] * rng.uniform(0.5, 1.0, (n, 3))))
    # zero axes: 1, 2 or 3 of the three scales exactly 0
    n = 48
    z = rng.uniform(1.0, 6.0, n)
    s = np.exp(rng.uniform(np.log(0.005), np.log(0.1), (n, 3)))
    nz = np.arange(n) % 3 + 1
    for i in range(n):
        s[i, rng.permutation(3)[: nz[i]]] = 0.0
    groups.append((np.concatenate([rng.uniform(-0.8, 0.8, (n, 2)) * np.array([tx, ty]) * z[:, None], z[:, None]], 1), s))
    xyz = np.concatenate([g[0] for g in groups]).astype(np.float32)   # float32 depths of the near group survive exactly
    scales = np.concatenate([g[1] for g in groups]).astype(np.float32)
    P = xyz.shape[0]
    opac = rng.uniform(0.05, 1.0, (P, 1)).astype(np.float32)
    return Cloud(xyz, scales, _random_quats(rng, P), opac, _sh_dc(rng, P, sh_degree), sh_degree), cam


def opacity_edge_cloud(seed: int = 0, stacks: int = 48):
    """Stacks of overlapping Gaussians at 320x240 -> (Cloud, Camera). Opacities: fp32(1/255) and its neighbours
    (the `alpha < 1/255` test and the culling early-out), 0.99 and above (the alpha clamp), and uniform ones; stack
    depths 2..160, so the T < 1e-4 stop falls at varied list positions (with two clamped layers T = 1e-4 exactly
    in real arithmetic)."""
    rng = np.random.default_rng(seed)
    W, H = 320, 240
    cam = look_at_camera((0, 0, -5), (0, 0, 0), (0, -1, 0), W, H, fovy_deg=50.0)
    o255 = np.float32(1.0 / 255.0)
    edge_lo = [np.nextafter(o255, np.float32(-1), dtype=np.float32), o255, np.nextafter(o255, np.float32(1), dtype=np.float32),
               np.float32(o255 * np.float32(1.0001)), np.float32(o255 * np.float32(1.01))]
    edge_hi = [np.float32(0.99), np.nextafter(np.float32(0.99), np.float32(1), dtype=np.float32),
               np.nextafter(np.float32(0.99), np.float32(0), dtype=np.float32), np.float32(0.995), np.float32(1.0)]
    depth_n = np.exp(rng.uniform(np.log(2), np.log(160), stacks)).astype(int)
    xyz, opac = [], []
    for s in range(stacks):
        n = depth_n[s]
        c = rng.uniform(-1.4, 1.4, 2) * np.array([1.0, 0.75])
        xyz.append(np.concatenate([c + rng.normal(0, 0.03, (n, 2)), rng.uniform(-1.0, 1.0, (n, 1))], 1))
        kind = rng.integers(0, 3, n)
        o = np.where(kind == 0, rng.choice(edge_lo, n), np.where(kind == 1, rng.choice(edge_hi, n), rng.uniform(0.05, 0.9, n)))
        opac.append(o)
    xyz = np.concatenate(xyz).astype(np.float32)
    P = xyz.shape[0]
    scales = np.exp(rng.uniform(np.log(0.02), np.log(0.12), (P, 3))).astype(np.float32)
    opac = np.concatenate(opac).astype(np.float32)[:, None]
    return Cloud(xyz, scales, _random_quats(rng, P), opac, _sh_dc(rng, P, 1), 1), cam


# ---- list-structure scenes ---------------------------------------------------------------------------------------
# Inputs that shape the per-tile instance lists rather than the splats: one tile holding more instances than a sort tile
# (4096) and than 2^16, depth keys shared by thousands of Gaussians, and instance counts at the kernels' block sizes.
# All three put the camera at the origin looking down +z, so the view depth of a Gaussian is its world z exactly.

def _origin_camera(W: int, H: int) -> Camera:
    return look_at_camera((0, 0, 0), (0, 0, 1), (0, -1, 0), W, H, fovx_deg=60.0)   # view (x, y, z) = world (-x, -y, z)


def _at_pixels(cam: Camera, px, py, z):
    """World centres that project to pixel coordinates (px, py) at view depth z (inverse of ndc2Pix and the
    projection of _origin_camera)."""
    W, H = cam.image_width, cam.image_height
    ndc_x = (2.0 * px + 1.0) / W - 1.0
    ndc_y = (2.0 * py + 1.0) / H - 1.0
    return np.stack([-ndc_x * cam.tanfovx * z, -ndc_y * cam.tanfovy * z, z], axis=1)


def _tiny_splats(rng, n):
    """Scales of 1e-5 (sub-pixel at depths 2..6): only the 0.3 px^2 dilation is left, and with the reference's 0.1 floor
    under the eigenvalue spread the radius is ceil(3 sqrt(0.3 + sqrt(0.1))) = 3 px."""
    return np.full((n, 3), 1e-5) * rng.uniform(0.8, 1.2, (n, 3))


def hotspot_cloud(P: int = 70_000, seed: int = 0, extra: int = 200):
    """One hot tile at 64x64 -> (Cloud, Camera). ``P`` near-isotropic sub-pixel Gaussians (radius 3 px) with centres
    uniform inside tile (1, 1) at depths 2..6 and opacities in [1.05/255, 3/255], so no pixel reaches the T < 1e-4 stop
    and every pixel of the tile walks the whole list: that tile's list holds about P instances (more than a sort tile of
    4096 and than 2^16 at the default P), and n_contrib reaches P. ``extra`` ordinary Gaussians elsewhere keep the other
    tiles from being empty. SH degree 0."""
    rng = np.random.default_rng(seed)
    cam = _origin_camera(64, 64)
    px, py = rng.uniform(16.0, 32.0, P), rng.uniform(16.0, 32.0, P)
    hot = _at_pixels(cam, px, py, rng.uniform(2.0, 6.0, P))
    other = _at_pixels(cam, rng.uniform(0.0, 64.0, extra), rng.uniform(0.0, 64.0, extra), rng.uniform(2.0, 6.0, extra))
    xyz = np.concatenate([hot, other]).astype(np.float32)
    scales = np.concatenate([_tiny_splats(rng, P), np.exp(rng.uniform(np.log(0.01), np.log(0.05), (extra, 3)))])
    opac = np.concatenate([rng.uniform(1.05 / 255.0, 3.0 / 255.0, P), rng.uniform(0.1, 0.9, extra)])
    n = P + extra
    return Cloud(xyz, scales.astype(np.float32), _random_quats(rng, n), opac.astype(np.float32)[:, None],
                 _sh_dc(rng, n, 0), 0), cam


def clone_rows(cloud: Cloud, seed: int = 0, fraction: float = 0.3) -> Cloud:
    """What GaussianEditor's densify_and_clone does to the list order: a random ``fraction`` of the rows copied 1..3
    times and the exact copies appended at the end (densification_postfix). A copy shares its original's depth key but
    sits far from it in index."""
    rng = np.random.default_rng(seed)
    P = cloud.means3D.shape[0]
    picked = rng.permutation(P)[: int(fraction * P)]
    rows = np.sort(np.repeat(picked, rng.integers(1, 4, picked.size)))
    cat = lambda a: np.ascontiguousarray(np.concatenate([a, a[rows]]))
    return Cloud(cat(cloud.means3D), cat(cloud.scales), cat(cloud.rotations), cat(cloud.opacities), cat(cloud.shs),
                 cloud.sh_degree)


def tied_depth_cloud(seed: int = 0, layer: int = 20_000, ordinary: int = 10_000):
    """A planar layer at 128x128 -> (Cloud, Camera): ``layer`` Gaussians at world z = 4 (one depth key, so equal keys
    span warps and CTAs of the depth sort) with their indices interleaved with ``ordinary`` Gaussians at depths 2..8, then
    clone_rows: a third of the rows copied 1..3 times and appended, so copies share keys with rows far away in index.
    Splats of a few pixels, opacities 0.05..0.5. SH degree 1."""
    rng = np.random.default_rng(seed)
    W = H = 128
    cam = _origin_camera(W, H)
    P = layer + ordinary
    z = np.where(np.arange(P) < layer, 4.0, rng.uniform(2.0, 8.0, P))
    z = z[rng.permutation(P)]
    xyz = _at_pixels(cam, rng.uniform(-8.0, W + 8.0, P), rng.uniform(-8.0, H + 8.0, P), z).astype(np.float32)
    xyz[:, 2] = z       # exactly 4.0 for the layer
    scales = np.exp(rng.uniform(np.log(0.005), np.log(0.03), (P, 3))).astype(np.float32)
    opac = rng.uniform(0.05, 0.5, (P, 1)).astype(np.float32)
    base = Cloud(xyz, scales, _random_quats(rng, P), opac, _sh_dc(rng, P, 1), 1)
    return clone_rows(base, seed=seed + 1), cam


ONE_TILE_COUNTS = (1, 2, 31, 32, 33, 127, 128, 129, 511, 512, 513, 4095, 4096, 4097, 8191, 8192, 8193)


def one_tile_cloud(P: int, W: int = 1024, H: int = 1024, seed: int = 0):
    """``P`` Gaussians that touch exactly one tile each -> (Cloud, Camera), so the instance count R equals P: sub-pixel
    splats (radius 3 px) whose centres lie 4..12 px into their tile. Depths are distinct (a permutation of an evenly
    spaced grid in 2..6). Half of the Gaussians go to four hot tiles, the rest to tiles drawn at random; at 1024x1024
    there are 4096 tiles, so both digits of the tile sort are used. SH degree 0. P in ONE_TILE_COUNTS puts R at and
    next to the multiples of the warp (32), the preprocess block (128), a warp's 512 sort slots and the sort tile
    (4096)."""
    rng = np.random.default_rng(seed)
    cam = _origin_camera(W, H)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    hot = rng.choice(gx * gy, 4, replace=False)
    tile = np.where(rng.uniform(size=P) < 0.5, hot[rng.integers(0, 4, P)], rng.integers(0, gx * gy, P))
    px = 16.0 * (tile % gx) + rng.uniform(4.0, 12.0, P)
    py = 16.0 * (tile // gx) + rng.uniform(4.0, 12.0, P)
    z = np.linspace(2.0, 6.0, P, dtype=np.float32)[rng.permutation(P)]
    xyz = _at_pixels(cam, px, py, z.astype(np.float64)).astype(np.float32)
    opac = rng.uniform(0.2, 0.9, (P, 1)).astype(np.float32)
    return Cloud(xyz, _tiny_splats(rng, P).astype(np.float32), _random_quats(rng, P), opac, _sh_dc(rng, P, 0), 0), cam


# ---- frame geometry ------------------------------------------------------------------------------------------------
def grid_camera(W: int, H: int) -> Camera:
    """_origin_camera with the 60-degree field of view across the frame's longer side (square pixels), so that frames
    one tile tall and one tile wide alike keep their centres away from the Jacobian clamp."""
    if W >= H:
        return _origin_camera(W, H)
    return look_at_camera((0, 0, 0), (0, 0, 1), (0, -1, 0), W, H, fovy_deg=60.0)


def _iso_scales(cam: Camera, xyz, r):
    """Isotropic scales that give splats centred at xyz (world = view up to signs, grid_camera) the integer radius r
    with half a pixel to spare: 3 sqrt(lambda_max) = r - 0.5. With J J^T = (f/z)^2 [[1 + u^2, uv], [uv, 1 + v^2]] the
    eigenvalues of s^2 J J^T + 0.3 are a + 0.3 and a (1 + u^2 + v^2) + 0.3 (a = (s f / z)^2), and the reference takes
    mid + sqrt(max(0.1, spread^2))."""
    f = cam.image_width / (2.0 * cam.tanfovx)
    z = xyz[:, 2]
    w2 = (xyz[:, 0] ** 2 + xyz[:, 1] ** 2) / z ** 2
    lam = ((np.asarray(r, np.float64) - 0.5) / 3.0) ** 2
    a = (lam - 0.3) / (1.0 + w2)
    small = a * w2 / 2.0 < np.sqrt(0.1)
    a = np.where(small, (lam - 0.3 - np.sqrt(0.1)) / (1.0 + w2 / 2.0), a)
    assert (a > 0).all()
    return np.sqrt(a) * z / f


def tile_grid_cloud(W: int, H: int, seed: int = 0, fill: int = 16384):
    """Isotropic Gaussians for a W x H frame of grid_camera -> (Cloud, Camera), laid out for the tile-binning tests:
      * one splat of radius 3..12 px in every tile row and one in every tile column, so every row and column of the tile
        grid holds instances;
      * ``fill`` splats of radius 3..24 px in the left 60 % of the frame, so R spans several 4096-instance sort tiles
        at every frame size while tiles in the right part stay empty (on grids of 50 tiles or more, at least two wide and
        tall);
      * three splats of radius 0.4 x the long side (at most 4000 px) and opacity 0.03..0.1 behind the others, each over
        hundreds of tiles along the long axis where the grid has them;
      * depths drawn from 97 values, so equal depth keys meet in many tiles.
    Centres sit at half-pixels and radii have half a pixel to spare, so fp32 rounding cannot move a tile edge. The rows
    are shuffled: kinds and tied depths interleave in index order. SH degree 0."""
    rng = np.random.default_rng(seed)
    cam = grid_camera(W, H)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    half = lambda lo, hi: np.floor(rng.uniform(lo, hi)) + 0.5          # half-pixel centres in [lo, hi)
    ty, tx = np.arange(gy), np.arange(gx)
    rows_py = half(16.0 * ty, np.minimum(16.0 * ty + 16.0, H))
    cols_px = half(16.0 * tx, np.minimum(16.0 * tx + 16.0, W))
    px = np.concatenate([half(np.zeros(gy), np.full(gy, W)), cols_px, half(np.zeros(fill), np.full(fill, 0.6 * W))])
    py = np.concatenate([rows_py, half(np.zeros(gx), np.full(gx, H)), half(np.zeros(fill), np.full(fill, H))])
    n_small = gy + gx
    r = np.concatenate([rng.integers(3, 13, n_small), rng.integers(3, 25, fill)])
    z = rng.choice(np.linspace(2.0, 8.0, 97), n_small + fill)
    opac = np.concatenate([rng.uniform(0.2, 0.8, n_small), rng.uniform(0.05, 0.5, fill)])
    long_side = max(W, H)
    rb = max(3, min(4000, int(0.4 * long_side)))
    big = 3
    bx = half(np.full(big, 0.25 * W), np.full(big, 0.35 * W))
    by = half(np.full(big, 0.4 * H), np.full(big, 0.6 * H))
    px, py = np.concatenate([px, bx]), np.concatenate([py, by])
    r = np.concatenate([r, np.full(big, rb)])
    z = np.concatenate([z, [8.5, 9.0, 9.5]])
    opac = np.concatenate([opac, rng.uniform(0.03, 0.1, big)])
    perm = rng.permutation(px.size)
    px, py, r, z, opac = px[perm], py[perm], r[perm], z[perm], opac[perm]
    P = px.size
    xyz = _at_pixels(cam, px, py, z)
    s = _iso_scales(cam, xyz, r)
    cloud = Cloud(xyz.astype(np.float32), np.repeat(s[:, None], 3, 1).astype(np.float32),
                  np.tile(np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), (P, 1)), opac.astype(np.float32)[:, None],
                  _sh_dc(rng, P, 0), 0)
    return cloud, cam


# ---- camera models -----------------------------------------------------------------------------------------------
# Cameras that look_at_camera cannot build: unequal focal lengths (PINHOLE intrinsics, resized frames), rolled and
# arbitrary rotations, very wide and very narrow fields of view, and a camera inside the cloud. Scenes are sampled in
# view space and carried to the world through the camera's inverse pose, so every pose sees its content.

def pinhole_camera(R_w2c, t, W: int, H: int, fx: float, fy: float) -> Camera:
    """GaussianEditor's ``Camera`` for the world-to-camera rotation ``R_w2c`` and translation ``t`` (camera coordinates
    R_w2c @ x + t) and focal lengths fx, fy in pixels: FoVx = focal2fov(fx, W), FoVy = focal2fov(fy, H), the
    projection of both FoVs, world_view_transform = W2C^T, full_proj_transform = world_view_transform @ P^T."""
    R = np.asarray(R_w2c, np.float64)
    t = np.asarray(t, np.float64)
    W2C = np.eye(4)
    W2C[:3, :3] = R
    W2C[:3, 3] = t
    tanx = math.tan(0.5 * (2.0 * math.atan(W / (2.0 * fx))))
    tany = math.tan(0.5 * (2.0 * math.atan(H / (2.0 * fy))))
    P = _projection(0.01, 100.0, tanx, tany)
    view_t = np.ascontiguousarray(W2C.astype(np.float32).T)
    proj_t = np.ascontiguousarray((view_t @ P.T).astype(np.float32))
    return Camera(H, W, float(tanx), float(tany), view_t, proj_t, (-R.T @ t).astype(np.float32))


def origin_aspect_focals(fx: float, fy: float, origin_w: int, origin_h: int, W: int, H: int):
    """The focal lengths in pixels of a ``W`` x ``H`` render of a PINHOLE intrinsic (fx, fy) of an ``origin_w`` x
    ``origin_h`` image, as GaussianEditor's COLMAP reader sets the FoVs when the aspect changes (readColmapCameras_hw:
    the longer side is cropped to the new aspect)."""
    aspect = H / W
    if origin_h / origin_w > aspect:           # shrink height
        fovy, fovx = 2 * math.atan(origin_w * aspect / (2 * fy)), 2 * math.atan(origin_w / (2 * fx))
    else:                                      # shrink width
        fovy, fovx = 2 * math.atan(origin_h / (2 * fy)), 2 * math.atan(origin_h / aspect / (2 * fx))
    return W / (2 * math.tan(fovx / 2)), H / (2 * math.tan(fovy / 2))


def random_rotation(rng, min_entry: float = 0.0) -> np.ndarray:
    """A uniformly random rotation matrix (QR of a Gaussian matrix), redrawn until every entry has |R_ij| >= min_entry."""
    while True:
        Q, Rr = np.linalg.qr(rng.standard_normal((3, 3)))
        Q = Q * np.sign(np.diag(Rr))[None, :]
        if np.linalg.det(Q) < 0:
            Q[:, 0] = -Q[:, 0]
        if np.abs(Q).min() >= min_entry:
            return Q


def _sh3(rng, P):
    shs = np.zeros((P, 16, 3), np.float32)
    shs[:, 0, :] = ((rng.uniform(size=(P, 3)) - 0.5) / SH_C0).astype(np.float32)
    k = 1
    for ell in range(1, 4):
        shs[:, k:k + 2 * ell + 1, :] = rng.standard_normal((P, 2 * ell + 1, 3)) * (0.15 / (1 + ell))
        k += 2 * ell + 1
    return shs


def _to_world(cam: Camera, xyz_view):
    """View-space points -> world space through the inverse of the camera's pose."""
    W2C = cam.viewmatrix.astype(np.float64).T
    R, t = W2C[:3, :3], W2C[:3, 3]
    return (np.asarray(xyz_view, np.float64) - t[None, :]) @ R


def view_space_cloud(cam: Camera, P: int, seed: int, near_frac: float = 0.1, clamp_frac: float = 0.2,
                     beyond_frac: float = 0.05) -> Cloud:
    """``P`` Gaussians sampled in ``cam``'s view space -> Cloud (world space), SH degree 3, random rotations:
      * ``near_frac`` at view depths in (0.2, 0.3], just beyond the near cut, centres inside the frame;
      * ``clamp_frac`` with |x/z|, |y/z| or both within 5 % of 1.3 tan(fov) (the Jacobian clamp), depths 0.5..20;
      * ``beyond_frac`` with centres 1.4..1.8 tan(fov) off axis in x or y (beyond the clamp), their scale large enough
        that the 3-sigma radius still reaches into the frame;
      * the rest inside the frame at depths 0.3..30.
    Projected sizes are 0.3..30 px per axis (in the larger focal length's pixels), opacities 0.05..0.95 (0.005..0.095
    beyond the clamp)."""
    rng = np.random.default_rng(seed)
    tan = np.array([cam.tanfovx, cam.tanfovy])
    f = max(cam.image_width / (2 * cam.tanfovx), cam.image_height / (2 * cam.tanfovy))
    n_near, n_clamp, n_beyond = int(near_frac * P), int(clamp_frac * P), int(beyond_frac * P)
    n_in = P - n_near - n_clamp - n_beyond
    z = np.concatenate([rng.uniform(0.2, 0.3, n_near), np.exp(rng.uniform(np.log(0.3), np.log(30.0), n_in)),
                        np.exp(rng.uniform(np.log(0.5), np.log(20.0), n_clamp + n_beyond))])
    z[:n_near] = np.maximum(z[:n_near], np.nextafter(np.float32(0.2), np.float32(1)))
    uv = rng.uniform(-0.9, 0.9, (P, 2)) * tan                         # x/z, y/z
    sgn = np.where(rng.uniform(size=(P, 2)) < 0.5, -1.0, 1.0)
    which = rng.integers(0, 3, P)                                     # x, y or both at the clamp / beyond
    axis = np.stack([which != 1, which != 0], 1)
    c0, c1 = n_near + n_in, n_near + n_in + n_clamp
    uv[c0:c1] = np.where(axis[c0:c1], sgn[c0:c1] * 1.3 * tan * rng.uniform(0.95, 1.05, (n_clamp, 2)), uv[c0:c1])
    off = rng.uniform(1.4, 1.8, (n_beyond, 2))
    uv[c1:] = np.where(axis[c1:], sgn[c1:] * off * tan, uv[c1:])
    sigma = np.exp(rng.uniform(np.log(0.3), np.log(30.0), (P, 1))) * np.exp(rng.uniform(-0.7, 0.7, (P, 3)))
    scales = sigma * z[:, None] / f
    # beyond: 3 sigma_min of the isotropic part at least 1.2x the distance from the centre to the frame's edge
    reach = (np.where(axis[c1:], off - 1.0, 0.0) * tan * z[c1:, None]).max(1)
    scales[c1:] = (1.2 * reach / 3.0)[:, None] * np.exp(rng.uniform(0.0, 0.5, (n_beyond, 3)))
    xyz = _to_world(cam, np.concatenate([uv * z[:, None], z[:, None]], 1))
    opac = rng.uniform(0.05, 0.95, (P, 1))
    opac[c1:] *= 0.1                     # the large off-frame splats: translucent, or together they hide the frame
    return Cloud(xyz.astype(np.float32), scales.astype(np.float32), _random_quats(rng, P), opac.astype(np.float32),
                 _sh3(rng, P), 3)


def camera_family(P: int = 3000, seed: int = 0) -> dict:
    """Named (Cloud, Camera) cases, every frame at most 640x480, seeded:
      aniso_0.5, aniso_2   fy / fx = 0.5 on 640x480 and 2 on 333x201, random poses;
      pinhole_resized      a 1297x840 PINHOLE intrinsic with fx != fy rendered at 512x512 (origin_aspect_focals);
      wide_120             fovx 120 degrees (tan 1.73), square pixels;
      tele_4               fovx 4 degrees (focal length 9160 px);
      roll_90              camera x = world +y, camera y = world -x: view[0] = 0, view[4] = 1;
      general              a random rotation with every entry at least 0.05 in magnitude;
      nadir                looking straight down world +y (look_at_camera with up (0, -1, 0) is degenerate there);
      inside               the eye at the centre of a bicycle_cloud of 2P (size 0.3), Gaussians in every direction, a few
                           of them large enough near the eye to cover the whole frame."""
    rng = np.random.default_rng(seed)
    out = {}

    def add(name, R, W, H, fx, fy, t=None):
        t = rng.normal(0.0, 2.0, 3) if t is None else t
        cam = pinhole_camera(R, t, W, H, fx, fy)
        out[name] = (view_space_cloud(cam, P, seed=int(rng.integers(1 << 30))), cam)

    add("aniso_0.5", random_rotation(rng), 640, 480, 520.0, 260.0)
    add("aniso_2", random_rotation(rng), 333, 201, 190.0, 380.0)
    add("pinhole_resized", random_rotation(rng), 512, 512, *origin_aspect_focals(1160.0, 1090.0, 1297, 840, 512, 512))
    fx = 320.0 / math.tan(math.radians(60.0))
    add("wide_120", random_rotation(rng), 640, 480, fx, fx)
    fx = 320.0 / math.tan(math.radians(2.0))
    add("tele_4", random_rotation(rng), 640, 480, fx, fx)
    add("roll_90", np.array([[0.0, 1, 0], [-1, 0, 0], [0, 0, 1]]), 640, 480, 500.0, 500.0)
    add("general", random_rotation(rng, min_entry=0.05), 640, 480, 560.0, 480.0)
    add("nadir", np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]]), 480, 360, 420.0, 420.0)
    # inside: eye at the origin of the bicycle cloud; eight large Gaussians just in front of it cover the frame
    cam = pinhole_camera(random_rotation(rng), np.zeros(3), 640, 480, 500.0, 450.0)
    base = bicycle_cloud(2 * P, seed=int(rng.integers(1 << 30)), size=0.3)
    n = 8
    big_view = np.concatenate([rng.uniform(-0.1, 0.1, (n, 2)), rng.uniform(0.4, 1.5, (n, 1))], 1)
    big = Cloud(_to_world(cam, big_view).astype(np.float32),
                (big_view[:, 2:] * rng.uniform(1.0, 2.0, (n, 3))).astype(np.float32), _random_quats(rng, n),
                rng.uniform(0.02, 0.1, (n, 1)).astype(np.float32), _sh3(rng, n), 3)
    out["inside"] = (Cloud(*(np.ascontiguousarray(np.concatenate([getattr(base, k), getattr(big, k)]))
                             for k in ("means3D", "scales", "rotations", "opacities", "shs")), 3), cam)
    return out


CONFIGS = {
    # name: (P, sh_degree, W, H)
    "c1": dict(P=10_000, sh_degree=0, W=256, H=256),
    "c2": dict(P=100_000, sh_degree=0, W=800, H=800),
    "c3": dict(P=1_000_000, sh_degree=3, W=1600, H=1200),
    "c4": dict(P=5_000_000, sh_degree=3, W=1920, H=1080),
    "c5": dict(P=500_000, sh_degree=3, W=512, H=512),
}


def make_config(name: str, P: int | None = None):
    """Returns (Cloud, [Camera, ...]) for a BASELINE.json config. ``P`` overrides the
    Gaussian count (used for bounded CPU samples and small parity cases)."""
    c = CONFIGS[name]
    P = c["P"] if P is None else P
    W, H = c["W"], c["H"]
    if name == "c1":
        return cube_cloud(P, 1, 0.03), [look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), W, H, fovy_deg=50.0)]
    if name == "c2":
        return cube_cloud(P, 2, 0.012), [look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), W, H, fovy_deg=50.0)]
    if name == "c3":
        return bicycle_cloud(P, 3), ring_cameras(8, 4.5, 15.0, W, H, 61.0)
    if name == "c4":
        return bicycle_cloud(P, 4), ring_cameras(8, 4.5, 15.0, W, H, 61.0)
    if name == "c5":
        return bicycle_cloud(P, 5, size=0.5), ring_cameras(48, 2.25, 15.0, W, H, 61.0)
    raise KeyError(name)


def make_config_cached(name: str, P: int | None = None, cache_dir: str = "/tmp"):
    """make_config with the cloud cached as .npy files under `cache_dir` (multi-process benches: the 5M-Gaussian cloud
    takes ~45 s to generate; ranks other than the first to arrive just load it). Cameras are always recomputed."""
    import os
    import time
    tag = f"gsr_synth_{name}_{CONFIGS[name]['P'] if P is None else P}"
    done = os.path.join(cache_dir, tag + ".done")
    lock = os.path.join(cache_dir, tag + ".lock")
    fields = ["means3D", "scales", "rotations", "opacities", "shs"]
    cams = None
    if not os.path.exists(done):
        try:
            fd = os.open(lock, os.O_CREAT | os.O_EXCL | os.O_WRONLY)
            os.close(fd)
            cloud, cams = make_config(name, P)
            for f in fields:
                np.save(os.path.join(cache_dir, f"{tag}_{f}.npy"), getattr(cloud, f))
            with open(done, "w") as fh:
                fh.write(str(cloud.sh_degree))
            return cloud, cams
        except FileExistsError:
            while not os.path.exists(done):
                time.sleep(0.5)
    with open(done) as fh:
        deg = int(fh.read())
    arrs = {f: np.load(os.path.join(cache_dir, f"{tag}_{f}.npy")) for f in fields}
    c = CONFIGS[name]
    small = make_config(name, 16)[1]  # cameras do not depend on P
    return Cloud(sh_degree=deg, **arrs), small
