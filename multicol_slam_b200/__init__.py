"""multicol_slam_b200 -- H100-native (sm_90a) feature hot path of MultiCol-SLAM behind a C ABI.

Only the path named in BASELINE.json's north_star lives here: csrc/ (CUDA kernels + libmcs_b200.so),
the ctypes mirror of the C ABI (api.py) and the synthetic-data helpers the tests and bench share."""
