"""
Drop-in mirror of the reference's DENSE fog (lib/LiDAR_fog_sim/SeeingThroughFog/tools/DatasetFoggification/):
`BetaRadomization(beta, seed=None, param_set='DENSE')` (beta_modification.py:5-114) and
`haze_point_cloud(pts_3D, beta_radomization, arguments)` (lidar_foggification.py:61-149), computed by the CUDA engine
(csrc/haze.cu).  Caller in the reference: DenseDataset.foggify, dense_dataset.py:977-985.

BetaRadomization draws its Fourier parameters from NumPy's global RandomState exactly as the reference does (seed given:
np.random.seed first); haze_point_cloud draws the rest of the cloud's randomness from the same global state, on the
device, and leaves it where the reference leaves it.  Outputs are the reference's: float64 rows with F + 1 columns
(label 0 stable, 1 cloud scatter, 2 random scatter), and for beta == 0 the tuple (rows with label 0, []).

Exactness (DESIGN.md §7.10): rows, labels, order and the generator state equal the reference's; float64 values within a
few ulp (CUDA's sin / exp are not glibc's).  The device's tan(y / x) is the correctly rounded float32; a host whose
float32 np.tan is not correctly rounded gives some rows a different beta field (pass `angle=` to replay it).
"""
import numpy as np
import torch

from ..engine import default_engine

SUPPORTED_SENSORS = ['Velodyne HDL-64E S2', 'Velodyne HDL-64E S3D']          # lidar_foggification.py:21-22
SENSOR_CONSTANTS = {'Velodyne HDL-64E S3D': (0.04, 0.45, 2),                 # (n, g, dmin), :76-84
                    'Velodyne HDL-64E S2': (0.05, 0.35, 2)}


class BetaRadomization:
    """beta_modification.py:5-114, the 'DENSE' parameter set (the one the dataset uses)."""

    def __init__(self, beta, seed=None, param_set='DENSE'):
        if param_set in ('DENSE_use_n_heights', 'DENSE_no_noise', 'CVL'):
            raise NotImplementedError(f'param_set {param_set!r}: only the DENSE parameter set is implemented')
        if seed is not None:
            np.random.seed(seed)
        self.noise_mean = 0.0
        self.noise_std = 0.0
        self.beta = beta
        magnitude, mhf, mvf = 0.05, 2, 5
        n_components = np.random.randint(6, 10)
        self.frequencies_angle = np.random.randint(1, mhf, size=n_components)
        self.frequencies_height = np.random.randint(0, mvf, size=n_components)
        self.offset_angle = np.random.uniform(0, 2 * np.pi, size=n_components)
        self.offset_height = np.random.uniform(0, 2 * np.pi, size=n_components)
        self.intensity_angle = np.random.uniform(0, magnitude / n_components, size=n_components)
        self.intensity_height = np.random.uniform(0, magnitude / n_components, size=n_components)

    def propagate_in_time(self, timestep):
        self.offset_angle += self.frequencies_angle * timestep / 10
        self.offset_height += self.frequencies_height * timestep / 10

    def fourier(self):
        """(n_components, 6) float64 rows (fa, fh, oa, oh, ih, ia): the parameters of the engine's beta field"""
        return np.stack([self.frequencies_angle, self.frequencies_height, self.offset_angle, self.offset_height,
                         self.intensity_height, self.intensity_angle], axis=1).astype(np.float64)


def haze_point_cloud(pts_3D, beta_radomization, arguments, *, engine=None, angle=None):
    """lidar_foggification.py:61-149 on one cloud (N, F >= 4), NumPy's global RandomState as the stream.  `arguments`
    needs sensor_type and fraction_random.  angle: optional float32 (N,) tangents to replay (see the module doc).
    Raises the reference's OverflowError('Range exceeds valid bounds') where its uniform draw of d_rand meets a NaN or
    infinite bound, NumPy's global state left after the lost draws as the reference leaves it."""
    sensor = getattr(arguments, 'sensor_type', None)
    if sensor not in SENSOR_CONSTANTS:
        # the reference leaves n, g, dmin None and fails in its first comparison
        raise TypeError(f"'>' not supported between instances of 'float' and 'NoneType' (sensor {sensor!r})")
    n_noise, gain, dmin = SENSOR_CONSTANTS[sensor]
    eng = engine or default_engine()
    pts = np.ascontiguousarray(pts_3D, dtype=np.float32)
    if pts.ndim != 2 or pts.shape[1] < 4:
        raise ValueError(f'pts_3D: expected (N, F >= 4) rows, got shape {pts.shape}')
    beta = float(beta_radomization.beta)
    # the tuple branch copies 4 columns into F + 1: the reference raises ValueError after its lost draws for F > 4
    bad_tuple = beta == 0.0 and pts.shape[1] != 4
    rows = pts[:, :4].copy() if bad_tuple else pts
    dev = torch.from_numpy(rows).to(eng.device)
    ang = None if angle is None else torch.from_numpy(np.ascontiguousarray(angle, np.float32)).to(eng.device)
    r = eng.haze_batch(dev, [0, rows.shape[0]], [beta], beta_radomization.fourier(), n_noise, gain, dmin,
                       float(arguments.fraction_random), angle=ang, out_dtype=torch.float64, label=True)
    if bad_tuple:
        raise ValueError(f'could not broadcast input array from shape ({int(r["counts"][0])},{pts.shape[1]}) into '
                         f'shape ({int(r["counts"][0])},4)')
    out = r['points'][:int(r['counts'][0])].cpu().numpy()
    return (out, []) if beta == 0.0 else out
