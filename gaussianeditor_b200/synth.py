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


# ---- magnitude scenes ----------------------------------------------------------------------------------------------
# Inputs at the magnitudes trained clouds reach: scales that vanish or overflow in fp32, screen radii past 2^24 and
# 2^31, 2-D covariances whose determinant is decided by rounding, scenes far from the origin or in other units.

def _fma32(a, b, c):
    """fp32 fma: the product of two floats is exact in fp64, the sum rounds once in fp64 and again to fp32 (the double
    rounding differs from the device only on an exact fp32 tie, which does not occur in these scenes)."""
    return np.asarray(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64), np.float32)


def preprocess_fp32(cloud: Cloud, cam: Camera) -> dict:
    """The forward preprocess's covariance, conic and radius arithmetic, operation for operation as the kernels (and the
    reference's CUDA build) round it at sm_90a (csrc/preprocess_fwd_body.inc), in numpy: the generators use it to put
    Gaussians on rounding edges. Keys: depth, means2D, cov3D [P,6], cov2 [P,3] (a, b, c), det, conic [P,3],
    radius_f (3 sqrt(lambda_max) rounded up, before the conversion), radius (saturated as cvt.rzi.s32.f32; 0 where
    the near cut or det == 0 culls)."""
    f32 = lambda a: np.asarray(a, np.float32)
    with np.errstate(all="ignore"):
        m, v, pm = f32(cloud.means3D), f32(cam.viewmatrix).reshape(-1), f32(cam.projmatrix).reshape(-1)
        x, y, z = m[:, 0], m[:, 1], m[:, 2]
        tp = lambda M, i: f32(_fma32(M[8 + i], z, _fma32(M[0 + i], x, np.float32(M[4 + i] * y))) + M[12 + i])
        t = [tp(v, 0), tp(v, 1), tp(v, 2)]
        hx, hy, hw = tp(pm, 0), tp(pm, 1), tp(pm, 3)
        pw = f32(1) / f32(hw + f32(1e-7))
        ndc = lambda p, S: f32(((p.astype(np.float64) + 1.0) * S - 1.0) * 0.5)
        means2D = np.stack([ndc(f32(hx * pw), cam.image_width), ndc(f32(hy * pw), cam.image_height)], 1)
        s = f32(cloud.scales)
        q = f32(cloud.rotations)
        r, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        xz, rx, rz, yy, zz = qx * qz, r * qx, r * qz, qy * qy, qz * qz
        e02, e20, e12 = _fma32(r, qy, xz), _fma32(-r, qy, xz), _fma32(qy, qz, -rx)
        e21, e01, e10 = _fma32(qy, qz, rx), _fma32(qx, qy, -rz), _fma32(qx, qy, rz)
        q00, q11, q22 = f32(yy + zz), _fma32(qx, qx, zz), _fma32(qx, qx, yy)
        R = [[f32(1) - (q00 + q00), e01 + e01, e02 + e02], [e10 + e10, f32(1) - (q11 + q11), e12 + e12],
             [e20 + e20, e21 + e21, f32(1) - (q22 + q22)]]
        Mm = [[s[:, k] * R[c][k] for k in range(3)] for c in range(3)]
        sig = lambda c, k: _fma32(Mm[k][2], Mm[c][2], _fma32(Mm[k][0], Mm[c][0], Mm[k][1] * Mm[c][1]))
        V = [sig(0, 0), sig(0, 1), sig(0, 2), sig(1, 1), sig(1, 2), sig(2, 2)]
        focal_x = f32(cam.image_width / f32(2.0 * f32(cam.tanfovx)))
        focal_y = f32(cam.image_height / f32(2.0 * f32(cam.tanfovy)))
        limx, limy = f32(1.3) * f32(cam.tanfovx), f32(1.3) * f32(cam.tanfovy)
        tx = np.minimum(limx, np.maximum(-limx, t[0] / t[2])) * t[2]
        ty = np.minimum(limy, np.maximum(-limy, t[1] / t[2])) * t[2]
        tz2 = t[2] * t[2]
        J00, J02 = focal_x / t[2], (-tx * focal_x) / tz2
        J11, J12 = focal_y / t[2], (-ty * focal_y) / tz2
        T00, T01, T02 = _fma32(v[2], J02, v[0] * J00), _fma32(v[6], J02, v[4] * J00), _fma32(v[10], J02, v[8] * J00)
        T10, T11, T12 = _fma32(v[2], J12, v[1] * J11), _fma32(v[6], J12, v[5] * J11), _fma32(v[10], J12, v[9] * J11)
        V00, V01, V02, V11, V12, V22 = V
        A00 = _fma32(T02, V02, _fma32(T00, V00, T01 * V01))
        A01 = _fma32(T12, V02, _fma32(T10, V00, T11 * V01))
        A10 = _fma32(T02, V12, _fma32(T00, V01, T01 * V11))
        A11 = _fma32(T12, V12, _fma32(T10, V01, T11 * V11))
        A20 = _fma32(T02, V22, _fma32(T00, V02, T01 * V12))
        A21 = _fma32(T12, V22, _fma32(T10, V02, T11 * V12))
        ca = f32(_fma32(T02, A20, _fma32(T00, A00, T01 * A10)) + f32(0.3))
        cb = _fma32(T02, A21, _fma32(T00, A01, T01 * A11))
        cc = f32(_fma32(T12, A21, _fma32(T10, A01, T11 * A11)) + f32(0.3))
        det = _fma32(ca, cc, -(cb * cb))
        dinv = f32(1) / det
        conic = np.stack([cc * dinv, cb * -dinv, ca * dinv], 1)
        mid = (ca + cc) * f32(0.5)
        disc = np.sqrt(np.fmax(f32(0.1), _fma32(mid, mid, -det)))
        lam = np.fmax(mid + disc, mid - disc)
        radius_f = np.ceil(f32(3) * np.sqrt(lam))
        rad = np.where(np.isnan(radius_f), 0, np.clip(np.nan_to_num(radius_f.astype(np.float64), posinf=2.0 ** 31),
                                                     -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)
        rad = np.where((t[2] > f32(0.2)) & (det != 0), rad, 0)
    return dict(depth=t[2], means2D=means2D, cov3D=np.stack(V, 1), cov2=np.stack([ca, cb, cc], 1), det=det,
                conic=conic, radius_f=radius_f, radius=rad)


def _pix_to_view(cam: Camera, px, py, z):
    """View-space point that projects to pixel (px, py) at view depth z (ndc from the tangents, as _at_pixels)."""
    vx = ((np.asarray(px, np.float64) + 0.5) * 2.0 / cam.image_width - 1.0) * cam.tanfovx * z
    vy = ((np.asarray(py, np.float64) + 0.5) * 2.0 / cam.image_height - 1.0) * cam.tanfovy * z
    return np.stack([vx, vy, np.asarray(z, np.float64)], -1)


MAGNITUDE_RADII = (16777215.0, 16777216.0, 16777218.0, 2147483520.0, 2147483648.0, 2147483904.0, 1e10, 1e12)


def magnitude_cloud(seed: int = 0):
    """Gaussians at the magnitudes trained clouds reach, 320x200 (a partial last tile row), camera at the origin looking
    down +z (view (x, y, z) = world (-x, -y, z) exactly), SH degree 3 -> (Cloud, Camera, groups), groups: name -> row
    indices. Every input is finite; only intermediates overflow or underflow. Front to back:
      opacity_*      opacities denormal, 0, fp32(1/255) and its two neighbours, 1; `sh_1e30` SH coefficients up to 1e30;
                     `clamp_zero` colours whose `+ 0.5` lands on exactly 0 in every channel (not clamped: the test is < 0);
      vanishing      isotropic scales 10^k, k = -30..-4: cov3D denormal or 0, the 2-D covariance the 0.3 dilation alone
                     (radius 3); `vanishing_mixed`: two such axes and one ordinary;
      cancel_tiny / cancel_negative   needles with axis ratios 1e4..1e8 and ~1e4 px long axes whose det a c - b^2
                     rounds to a small positive value (a conic of 1e3 and more) and below 0 (power > 0 almost everywhere:
                     binned, hardly ever blended); `cancel_zero`: needles with one non-zero axis whose det is exactly 0
                     (culled), built as described below;
      radius_edge    isotropic splats with 3 sqrt(lambda_max) = MAGNITUDE_RADII in fp32: just below, on and above 2^24,
                     2^31 - 1 (2147483520, then 2^31 and 2147483904, which saturate to INT_MAX) and beyond;
      overflow       isotropic scales 1e12 .. 1.8e19 (cov3D stays finite, sqrt(FLT_MAX) = 1.84e19): the 2-D covariance
                     reaches inf from 1e17 on, the conic is NaN and alpha = fminf(0.99, NaN) = 0.99 over the whole grid;
                     `overflow_rotated`: anisotropic and rotated, b = +-inf or NaN as well.
    The camera's tangents are 0.5 and 0.3125, so focal_x = focal_y = 320 exactly. Those far-back overflow splats are placed where no row of the scene's cov2 diagonal becomes NaN: a NaN radius converts
    to 0 and leaves the reference's tile count without instances (its instance slots unwritten)."""
    rng = np.random.default_rng(seed)
    W, H = 320, 200
    # tan(fovx / 2) = 0.5 and tan(fovy / 2) = 0.3125 exactly: focal_x = focal_y = 320 in fp32 (cancel_zero needs both)
    cam = look_at_camera((0, 0, 0), (0, 0, 1), (0, -1, 0), W, H, fovx_deg=math.degrees(2.0 * math.atan(0.5)))
    fx = W / (2.0 * cam.tanfovx)
    rows, groups = [], {}

    def add(name, view_xyz, scales, quats, opac, shs=None):
        n = len(scales)
        start = sum(len(r[1]) for r in rows)
        groups[name] = np.arange(start, start + n)
        world = np.asarray(view_xyz, np.float64) * np.array([-1.0, -1.0, 1.0])
        sh = _sh3(rng, n) if shs is None else shs
        rows.append((world.astype(np.float32), np.asarray(scales, np.float32), np.asarray(quats, np.float32),
                     np.asarray(opac, np.float32).reshape(n, 1), sh.astype(np.float32)))

    def on_frame(n, z0, z1):
        z = rng.uniform(z0, z1, n)
        return _pix_to_view(cam, rng.uniform(8, W - 8, n), rng.uniform(8, H - 8, n), z)

    # colour and opacity extremes (front): splats of 4..10 px
    o255 = np.float32(1.0 / 255.0)
    ops = [np.float32(1e-40), np.float32(1e-45), np.float32(0.0), np.nextafter(o255, np.float32(0)), o255,
           np.nextafter(o255, np.float32(1)), np.float32(1.0)]
    names = ["opacity_denormal", "opacity_denormal_min", "opacity_zero", "opacity_255_below", "opacity_255",
             "opacity_255_above", "opacity_one"]
    for nm, o in zip(names, ops):
        n = 4
        p = on_frame(n, 1.0, 2.0)
        add(nm, p, (p[:, 2:] * rng.uniform(4, 10, (n, 3)) / fx), _random_quats(rng, n), np.full(n, o))
    n = 8
    p = on_frame(n, 1.0, 2.0)
    sh = _sh3(rng, n)
    sh[:, :, :] *= np.float32(10.0) ** rng.integers(20, 31, (n, 16, 1))        # up to 1e30
    add("sh_1e30", p, p[:, 2:] * rng.uniform(3, 8, (n, 3)) / fx, _random_quats(rng, n), rng.uniform(0.3, 0.9, n), sh)
    # clamp_zero: DC only, fp32(SH_C0) * sh0 rounds to exactly -0.5, so the colour is -0.5 + 0.5 = +0 in every channel
    c0 = np.float32(SH_C0)
    cand = np.float32(-0.5 / SH_C0) + np.arange(-8, 9).astype(np.float32) * np.spacing(np.float32(-0.5 / SH_C0))
    sh0 = cand[(c0 * cand) == np.float32(-0.5)]
    assert sh0.size, "no fp32 coefficient with SH_C0 * c == -0.5"
    n = 6
    p = on_frame(n, 1.0, 2.0)
    sh = np.zeros((n, 16, 3), np.float32)
    sh[:, 0, :] = sh0[0]
    add("clamp_zero", p, p[:, 2:] * rng.uniform(3, 8, (n, 3)) / fx, _random_quats(rng, n), rng.uniform(0.3, 0.9, n), sh)
    # vanishing
    k = np.arange(-30, -3)
    n = k.size
    p = on_frame(n, 2.0, 5.0)
    add("vanishing", p, np.repeat((10.0 ** k)[:, None], 3, 1), _random_quats(rng, n), rng.uniform(0.3, 0.9, n))
    p = on_frame(n, 2.0, 5.0)
    s = np.repeat((10.0 ** k)[:, None], 3, 1)
    s[np.arange(n), rng.integers(0, 3, n)] = p[:, 2] * rng.uniform(3, 8, n) / fx
    add("vanishing_mixed", p, s, _random_quats(rng, n), rng.uniform(0.3, 0.9, n))
    # cancelling determinant: needles in the image plane (rotation about the view axis, tilt <= 2 degrees)
    N = 20000
    p = on_frame(N, 8.0, 12.0)
    s_long = 1e4 * p[:, 2] / fx
    ratio = 10.0 ** rng.uniform(4, 8, N)
    s = np.stack([s_long, s_long / ratio, s_long / ratio * rng.uniform(0.5, 2.0, N)], 1)
    q = _quat_mul(_axis_quats((0, 0, 1), rng.uniform(0, np.pi, N)), _axis_quats((0, 1, 0), np.radians(rng.uniform(-2, 2, N))))
    trial = Cloud((p * np.array([-1.0, -1.0, 1.0])).astype(np.float32), s.astype(np.float32), q.astype(np.float32),
                  np.ones((N, 1), np.float32), np.zeros((N, 16, 3), np.float32), 3)
    f = preprocess_fp32(trial, cam)
    det, cmax = f["det"], np.abs(f["conic"]).max(1)
    pick = {"cancel_tiny": np.flatnonzero((det > 0) & (cmax >= 1e3))[:8], "cancel_negative": np.flatnonzero(det < 0)[:8]}
    for nm, idx in pick.items():
        add(nm, p[idx], s[idx], q[idx], rng.uniform(0.2, 0.6, idx.size))
    # cancel_zero: with fma the determinant is a*c - round(b^2) exactly, 0 only if a*c fits in fp32. A needle with one
    # non-zero axis on the optical axis (J02 = J12 = 0) under an unnormalised quaternion (r, 0, 0, z) with
    # 1 - 2 z^2 == 2 r z in fp32 has V00 = V11 = V01 = (s R00)^2; with s R00 = 2^k and view depth 320 / 2^j the three
    # entries of the 2-D covariance are all 2^24 (the 0.3 rounds away), and det = 2^48 - 2^48 = 0
    zq = (np.float32(math.sin(math.pi / 8)).view(np.int32) + np.arange(-60, 61)).astype(np.int32).view(np.float32)
    rq = (np.float32(math.cos(math.pi / 8)).view(np.int32) + np.arange(-60, 61)).astype(np.int32).view(np.float32)
    Z, Rq = np.meshgrid(zq, rq)
    R00 = np.float32(1) - (Z * Z + Z * Z)
    eq = R00 == (Rq * Z) + (Rq * Z)
    zs, rs, rho = Z[eq], Rq[eq], R00[eq]
    for i, (depth, m) in enumerate(((10.0, 128.0), (20.0, 256.0), (40.0, 512.0))):
        sx = (np.float32(m / rho[i]).view(np.int32) + np.arange(-20, 21)).astype(np.int32).view(np.float32)
        n = sx.size
        tr = Cloud(np.tile(np.array([[0, 0, depth]], np.float32), (n, 1)),
                   np.stack([sx, np.zeros(n, np.float32), np.zeros(n, np.float32)], 1),
                   np.tile(np.array([[rs[i], 0, 0, zs[i]]], np.float32), (n, 1)), np.ones((n, 1), np.float32),
                   np.zeros((n, 16, 3), np.float32), 3)
        hit = np.flatnonzero(preprocess_fp32(tr, cam)["det"] == 0)
        assert hit.size, "no exactly cancelling determinant"
        sx = sx[hit[:1]]
        add("cancel_zero" if i == 0 else f"cancel_zero_{i}", np.array([[0.0, 0.0, depth]]),
            np.array([[sx[0], 0.0, 0.0]]), np.array([[rs[i], 0, 0, zs[i]]]), np.array([0.5]))
    groups["cancel_zero"] = np.concatenate([groups.pop(k) for k in ("cancel_zero", "cancel_zero_1", "cancel_zero_2")])
    # radius edges: isotropic splats at depth 30..40, the scale stepped by fp32 ulps until 3 sqrt(lambda_max) hits the
    # target (the rounding of det and of mid^2 - det makes the radius jump by up to ~1e3 between neighbouring scales, so
    # a target may need a few positions); beyond 2^31 the scale is only sized
    n = len(MAGNITUDE_RADII)
    p = np.zeros((n, 3))
    s = np.zeros(n, np.float32)
    steps = np.arange(-20000, 20001)
    for i, target in enumerate(MAGNITUDE_RADII):
        for attempt in range(40):
            p[i] = on_frame(1, 30.0, 40.0)[0]

            def radius_f(cs):
                m = len(cs)
                tr = Cloud(np.repeat((p[i:i + 1] * np.array([-1.0, -1.0, 1.0])).astype(np.float32), m, 0),
                           np.repeat(np.asarray(cs, np.float32)[:, None], 3, 1),
                           np.tile(np.array([[1, 0, 0, 0]], np.float32), (m, 1)), np.ones((m, 1), np.float32),
                           np.zeros((m, 16, 3), np.float32), 3)
                return preprocess_fp32(tr, cam)["radius_f"].astype(np.float64)
            s[i] = np.float32(target / 3.0 * p[i, 2] / fx)
            if target > 2.0 ** 32:
                break
            s0 = np.float32(s[i] * target / radius_f([s[i]])[0])     # the off-axis Jacobian term, removed
            cs = (s0.view(np.int32) + steps).astype(np.int32).view(np.float32)
            hit = np.flatnonzero(radius_f(cs) == target)
            if hit.size:
                s[i] = cs[hit[0]]
                break
        else:
            raise AssertionError(("no scale reaches radius", target))
    add("radius_edge", p, np.repeat(s[:, None], 3, 1), np.tile([1.0, 0, 0, 0], (n, 1)), rng.uniform(0.05, 0.15, n))
    # overflow (back): isotropic, identity rotation (cov3D diagonal), and rotated anisotropic ones kept where the
    # cov2 diagonal stays free of NaN
    s_iso = np.array([1e12, 1e14, 1e16, 1e17, 3e17, 1e18, 3e18, 1e19, 1.8e19])
    n = s_iso.size
    p = on_frame(n, 60.0, 90.0)
    add("overflow", p, np.repeat(s_iso[:, None], 3, 1), np.tile([1.0, 0, 0, 0], (n, 1)), rng.uniform(0.2, 0.9, n))
    N = 4000
    p = on_frame(N, 60.0, 90.0)
    s = 10.0 ** rng.uniform(16.5, 19.2, (N, 3))
    q = _random_quats(rng, N)
    trial = Cloud((p * np.array([-1.0, -1.0, 1.0])).astype(np.float32), s.astype(np.float32), q,
                  np.ones((N, 1), np.float32), np.zeros((N, 16, 3), np.float32), 3)
    f = preprocess_fp32(trial, cam)
    ok = ~np.isnan(f["cov2"][:, 0]) & ~np.isnan(f["cov2"][:, 2]) & np.isfinite(f["cov3D"]).all(1)
    b_inf, b_nan = ok & np.isinf(f["cov2"][:, 1]), ok & np.isnan(f["cov2"][:, 1])
    b_fin = ok & np.isfinite(f["cov2"][:, 1]) & np.isinf(f["cov2"][:, [0, 2]]).any(1)
    idx = np.concatenate([np.flatnonzero(b_inf)[:4], np.flatnonzero(b_nan)[:2], np.flatnonzero(b_fin)[:4]])
    add("overflow_rotated", p[idx], s[idx], q[idx], rng.uniform(0.2, 0.9, idx.size))
    cloud = Cloud(*(np.ascontiguousarray(np.concatenate([r[i] for r in rows])) for i in range(5)), 3)
    return cloud, cam, groups


def rescaled_patch(kind: str, factor: float, seed: int = 0, P: int = 3000):
    """A bicycle_cloud patch (SH degree 3) and a look-at camera, 240x160, moved together: kind "translate" adds
    (factor, -factor/2, factor/3) to every centre, to the eye and to its target, kind "scale" multiplies centres, scales and
    the eye by factor ("scale" with factor 1 is the patch itself). Fifty Gaussians sit straight in front of the eye at view depths from 1e-6
    to 60 (log-uniform), so at every factor some fall on each side of the near cut (view z = 0.2, not scale-invariant,
    nor is the 1e-7 in the projection's w) -> (Cloud, Camera)."""
    rng = np.random.default_rng(seed)
    base = bicycle_cloud(P, seed=seed + 1, size=0.5)
    eye = np.array([0.0, -0.8, -6.0])
    n = 50
    z = 10.0 ** rng.uniform(-6, np.log10(60.0), n)
    fwd = -eye / np.linalg.norm(eye)
    near = eye + z[:, None] * fwd + rng.normal(0, 1, (n, 3)) * (0.05 * z)[:, None]
    means = np.concatenate([base.means3D.astype(np.float64), near])
    scales = np.concatenate([base.scales.astype(np.float64), (0.01 * z)[:, None] * rng.uniform(0.5, 1.5, (n, 3))])
    extra = Cloud(near.astype(np.float32), scales[-n:].astype(np.float32), _random_quats(rng, n),
                  rng.uniform(0.02, 0.3, (n, 1)).astype(np.float32), _sh3(rng, n), 3)
    rot = np.concatenate([base.rotations, extra.rotations])
    opac = np.concatenate([base.opacities, extra.opacities])
    shs = np.concatenate([base.shs, extra.shs])
    target = np.zeros(3)
    if kind == "translate":
        t = factor * np.array([1.0, -0.5, 1.0 / 3.0])
        means, eye, target = means + t, eye + t, target + t
    elif kind == "scale":
        means, scales, eye = means * factor, scales * factor, eye * factor
    else:
        raise ValueError(kind)
    cam = look_at_camera(eye, target, (0, -1, 0), 240, 160, fovx_deg=55.0)
    return Cloud(means.astype(np.float32), scales.astype(np.float32), rot, opac, shs, 3), cam


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
