"""
Camera calibrations of the SeeingThroughFog (DENSE) rigs, HDL-64 and VLP-32, used by the camera field-of-view filters.

Calibration DATA of the dataset (the values the reference ships as lib/OpenPCDet/data/dense/calib_hdl64.txt and
calib_vlp32.txt, lines P2 / R0_rect / Tr_velo_to_cam; the two share P2 and R0), parsed to float32 exactly as lib/OpenPCDet/pcdet/utils/calibration_kitti.py:5-20
does (np.array(strings, dtype=np.float32)).  Consumed by tools/snowfall/simulation.py:532-540 and by the dataset's
FOV_POINTS_ONLY key through get_calib(sensor_type) (dense_dataset.py:30-33,689-711).
"""
import numpy as np

_P2 = ('2355.722801 0.0 988.138054 0.0 0.0 2355.722801 508.051838 0.0 0.0 0.0 1.0 0.0')
_R0 = ('1.0 0.0 0.0 0.0 1.0 0.0 0.0 0.0 1.0')
_V2C = ('0.008165559536184884 -0.9999654854673377 -0.0015334638999611712 0.08749686458036277 '
        '-0.007155442920435107 0.001475045689574084 -0.9999733115822772 -0.4164032939864676 '
        '0.9999410599000692 0.008176314223727743 -0.007143151380269915 -0.6955577980059064')
_V2C_VLP32 = ('0.019182254004378424 -0.999814941483157 -0.001457366920958193 0.09446519283833317 '
              '0.004827824788246401 0.0015502436327140112 -0.9999871443436125 -0.31301523548185484 '
              '0.9998043474796083 0.019174971491765617 0.004856668525282896 -0.29075840489873284')


def parse_calib_text(path):
    """Read a KITTI-style calib file with P2 / R0_rect / Tr_velo_to_cam on lines 3, 5, 6 (calibration_kitti.py:5-20)."""
    with open(path) as f:
        lines = f.readlines()
    return {'P2': np.array(lines[2].strip().split(' ')[1:], dtype=np.float32).reshape(3, 4),
            'R0': np.array(lines[4].strip().split(' ')[1:], dtype=np.float32).reshape(3, 3),
            'V2C': np.array(lines[5].strip().split(' ')[1:], dtype=np.float32).reshape(3, 4),
            'img_shape': (1024, 1920)}


STF_HDL64_CAMERA = {
    'P2': np.array(_P2.split(' '), dtype=np.float32).reshape(3, 4),
    'R0': np.array(_R0.split(' '), dtype=np.float32).reshape(3, 3),
    'V2C': np.array(_V2C.split(' '), dtype=np.float32).reshape(3, 4),
    'img_shape': (1024, 1920),          # simulation.py:536
}

STF_VLP32_CAMERA = {
    'P2': np.array(_P2.split(' '), dtype=np.float32).reshape(3, 4),
    'R0': np.array(_R0.split(' '), dtype=np.float32).reshape(3, 3),
    'V2C': np.array(_V2C_VLP32.split(' '), dtype=np.float32).reshape(3, 4),
    'img_shape': (1024, 1920),
}

# get_calib(sensor_type) of dense_dataset.py:30-33, by the dataset's sensor names
DENSE_CAMERAS = {'hdl64': STF_HDL64_CAMERA, 'vlp32': STF_VLP32_CAMERA}
