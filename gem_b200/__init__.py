"""gem_b200 -- H100-native (sm_90a) replacement for GEM's point-cloud -> elevation-grid fusion
hot path (the reference's libgpu.so).  The product is the CUDA library behind include/gem_b200.h;
this package is its Python host mirror used by tests and benchmarks."""
from ._lib import GemError, GemFrame, GemSensorModel, load  # noqa: F401
from .elevation_map import (CameraImage, ElevationMap, LaserSensorProcessor, PerfectSensorProcessor,  # noqa: F401
                            PointCloud2Layout, RosHeader, StereoSensorProcessor, StructuredLightSensorProcessor, make_frame)
