"""Host-side, load-time map pipeline and lookup tables (numpy; runs once per map).

Restates the reference's load-time code so that the device tables are bit-identical to what the
reference's ScanSimulator2D / RaceCar hold:
  load_map            <- laser_models.py:383-427 ScanSimulator2D.set_map (+ :40-53 get_dt)
  angle_lut           <- laser_models.py:379-381 (linspace(0, 2pi, theta_dis) INCLUSIVE of 2pi)
  beam_tables         <- base_classes.py:122-158 RaceCar.__init__
  theta_index_increment <- laser_models.py:367-368
The third-party calls are the same ones the reference makes (PIL decode, yaml, scipy EDT).
"""
import math
import os

import numpy as np

PARAM_KEYS = ['mu', 'C_Sf', 'C_Sr', 'lf', 'lr', 'h', 'm', 'I', 's_min', 's_max', 'sv_min', 'sv_max',
              'v_switch', 'a_max', 'v_min', 'v_max', 'width', 'length']

# f110_env.py:130
DEFAULT_PARAMS = {'mu': 1.0489, 'C_Sf': 4.718, 'C_Sr': 5.4562, 'lf': 0.15875, 'lr': 0.17145, 'h': 0.074,
                  'm': 3.74, 'I': 0.04712, 's_min': -0.4189, 's_max': 0.4189, 'sv_min': -3.2,
                  'sv_max': 3.2, 'v_switch': 7.319, 'a_max': 9.51, 'v_min': -5.0, 'v_max': 20.0,
                  'width': 0.31, 'length': 0.58}

MAPS_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'maps')


def params_vector(params):
    return np.array([float(params[k]) for k in PARAM_KEYS], dtype=np.float64)


def resolve_map_path(map_name):
    """f110_env.py:108-120: bundled names resolve inside the package, anything else is `<name>.yaml`."""
    if map_name in ('berlin', 'skirk', 'levine', 'vegas', 'stata_basement', 'example_map'):
        return os.path.join(MAPS_DIR, map_name + '.yaml')
    return map_name + '.yaml'


class HostMap(object):
    """What ScanSimulator2D holds after set_map, as numpy (fp64 DT, metadata)."""

    def __init__(self, dt, resolution, origin):
        self.dt = np.ascontiguousarray(dt, dtype=np.float64)
        self.height, self.width = self.dt.shape
        self.resolution = float(resolution)
        self.orig_x = float(origin[0])
        self.orig_y = float(origin[1])
        self.orig_s = float(np.sin(origin[2]))
        self.orig_c = float(np.cos(origin[2]))
        self.dt_oob = float(self.dt[-1, -1])      # xy_2_rc's (-1,-1) wraps to the last cell
        m, e = math.frexp(self.resolution)
        self.fast_path = int(m == 0.5 and self.orig_c == 1.0 and self.orig_s == 0.0)

    @classmethod
    def meta(cls, height, width, resolution, origin, dt_oob):
        """Metadata only, for a map whose table exists on the device alone (`DeviceMap.from_device_dt`)."""
        self = cls.__new__(cls)
        self.dt = None
        self.height, self.width = int(height), int(width)
        self.resolution = float(resolution)
        self.orig_x, self.orig_y = float(origin[0]), float(origin[1])
        self.orig_s, self.orig_c = float(np.sin(origin[2])), float(np.cos(origin[2]))
        self.dt_oob = float(dt_oob)
        m, e = math.frexp(self.resolution)
        self.fast_path = int(m == 0.5 and self.orig_c == 1.0 and self.orig_s == 0.0)
        return self


def code_table(values, ncodes=255):
    """Lossless byte coding of a DT grid: code = rank of the cell value among the `ncodes` smallest distinct
    values, 255 = escape.  Returns (codes uint8 [H,W], lut float64 [256]); lut[code] == value bit-exactly."""
    uniq = np.unique(values)
    small = uniq[:ncodes]
    lut = np.full((256,), np.nan)
    lut[:small.size] = small
    pos = np.searchsorted(small, values)
    pos_c = np.minimum(pos, small.size - 1)
    exact = (pos < small.size) & (small[pos_c] == values)
    codes = np.where(exact, pos_c, 255).astype(np.uint8)
    return np.ascontiguousarray(codes), lut


def load_bitmap(map_path, map_ext):
    """Image + yaml part of ScanSimulator2D.set_map (laser_models.py:397-422): returns (bitmap {0,255} fp64 with
    row 0 = image bottom, resolution, origin)."""
    import yaml
    from PIL import Image
    map_img_path = os.path.splitext(map_path)[0] + map_ext
    img = np.array(Image.open(map_img_path).transpose(Image.FLIP_TOP_BOTTOM)).astype(np.float64)
    img[img <= 128.] = 0.
    img[img > 128.] = 255.
    with open(map_path, 'r') as f:
        meta = yaml.safe_load(f)
    return img, meta['resolution'], meta['origin']


def load_map(map_path, map_ext):
    """Host pipeline, exactly the reference's: scipy EDT (laser_models.py:40-53, :425)."""
    from scipy.ndimage import distance_transform_edt as edt
    img, resolution, origin = load_bitmap(map_path, map_ext)
    return HostMap(resolution * edt(img), resolution, origin)


def device_edt(bitmap, resolution, device):
    """resolution * distance_transform_edt(bitmap) computed on the GPU (C ABI f110_edt); returns an fp64 CUDA
    tensor bit-identical to the scipy result."""
    import torch
    from . import _native as nat
    occ = torch.from_numpy(np.ascontiguousarray(bitmap == 0).astype(np.uint8)).to(device)
    H, W = occ.shape
    scratch = torch.empty((H, W), dtype=torch.int32, device=device)
    out = torch.empty((H, W), dtype=torch.float64, device=device)
    nat.check(nat.lib().f110_edt(nat.ptr(occ), H, W, float(resolution), nat.ptr(scratch), nat.ptr(out), None,
                                 torch.cuda.current_stream(device).cuda_stream))
    return out


def load_map_device_edt(map_path, map_ext, device):
    """Same map, with the distance transform done on the device (exact, same table as scipy's)."""
    img, resolution, origin = load_bitmap(map_path, map_ext)
    dt = device_edt(img, resolution, device)
    return HostMap(dt.cpu().numpy(), resolution, origin)


def angle_lut(theta_dis=2000):
    theta_arr = np.linspace(0.0, 2 * np.pi, num=theta_dis)
    return np.sin(theta_arr), np.cos(theta_arr)


def theta_index_increment(num_beams, fov, theta_dis=2000):
    angle_increment = fov / (num_beams - 1)
    return theta_dis * angle_increment / (2. * np.pi)


def beam_tables(num_beams, fov, params):
    scan_ang_incr = fov / (num_beams - 1)
    cosines = np.zeros((num_beams,))
    scan_angles = np.zeros((num_beams,))
    side_distances = np.zeros((num_beams,))
    dist_sides = params['width'] / 2.
    dist_fr = (params['lf'] + params['lr']) / 2.
    for i in range(num_beams):
        angle = -fov / 2. + i * scan_ang_incr
        scan_angles[i] = angle
        cosines[i] = np.cos(angle)
        if angle > 0:
            if angle < np.pi / 2:
                to_side, to_fr = dist_sides / np.sin(angle), dist_fr / np.cos(angle)
            else:
                to_side, to_fr = dist_sides / np.cos(angle - np.pi / 2.), dist_fr / np.sin(angle - np.pi / 2.)
        else:
            if angle > -np.pi / 2:
                to_side, to_fr = dist_sides / np.sin(-angle), dist_fr / np.cos(-angle)
            else:
                to_side, to_fr = dist_sides / np.cos(-angle - np.pi / 2), dist_fr / np.sin(-angle - np.pi / 2)
        side_distances[i] = min(to_side, to_fr)
    return scan_angles, cosines, side_distances


def load_waypoints(csv_path=None):
    """examples/example_waypoints.csv (';'-delimited, 3 header rows; cols x=1, y=2, psi=3).  Returns start
    poses (x, y, psi + pi/2) — the CSV heading is measured from +y (config_example_map.yaml:11-22)."""
    if csv_path is None:
        csv_path = os.path.join(MAPS_DIR, 'example_waypoints.csv')
    wp = np.loadtxt(csv_path, delimiter=';', skiprows=3)
    return np.stack([wp[:, 1], wp[:, 2], wp[:, 3] + np.pi / 2], axis=1)
