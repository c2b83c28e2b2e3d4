"""visualdet3d_b200 — GPU-native (H100, sm_90a) inference forward for visualDet3D's dense 3D-detection hot path.

Only what the path needs lives here: ``csrc/`` (hand-written CUDA kernels behind a C ABI, ``include/vd3d_b200.h``),
the ctypes binding (``_lib``), the host-side mirror of the reference's registry / detector interface
(``registry``, ``detectors``), the two op modules the reference builds under make.sh (``ops.dcn``, ``ops.iou3d``)
and the synthetic data generators used by the bench and the tests (``synth``).
"""
__version__ = "0.1.0"
