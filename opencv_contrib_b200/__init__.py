"""opencv_contrib_b200 -- H100-native (sm_90a) re-implementation of the dense optical-flow path
of opencv_contrib's cudaoptflow module (cv::cuda::DenseOpticalFlow family).

Only what the hot path needs lives here:
  csrc/            hand-written CUDA kernels + C++ host engines + the C ABI (libb200flow.so)
  _lib.py          ctypes binding of include/b200flow.h
  cudaoptflow.py   Python mirror of the reference's generated bindings
                   (cv2.cuda.OpticalFlowDual_TVL1_create(...).calc(I0, I1, flow, stream))
  batch.py         batched frame-pair front end, one process per GPU (torch.distributed / NCCL)
  video.py         consecutive-frame front end (one upload per frame, warm start, 3-stream pipeline)
  frames.py        interpolateFrames, the consumer right after the solvers
  flowio.py        Middlebury .flo files + the reference's error statistics
  superres.py      superres's BTV-L1 video super-resolution and its four CUDA optical-flow wrappers
  cudaimgproc.py   cudaimgproc's corner responses and GoodFeaturesToTrack detector
  lkpyramid.py     the video module's calcOpticalFlowPyrLK, buildOpticalFlowPyramid and SparsePyrLKOpticalFlow
  optflowgf.py     the video module's calcOpticalFlowFarneback and FarnebackOpticalFlow
"""
from .cudaoptflow import (  # noqa: F401
    DenseOpticalFlow,
    OpticalFlowDual_TVL1,
    FarnebackOpticalFlow,
    BroxOpticalFlow,
    DensePyrLKOpticalFlow,
    DeepFlowOpticalFlow,
    DISOpticalFlow,
    VariationalRefinement,
    OpticalFlowDual_TVL1_create,
    FarnebackOpticalFlow_create,
    BroxOpticalFlow_create,
    DensePyrLKOpticalFlow_create,
    createOptFlow_DeepFlow,
    DISOpticalFlow_create,
    VariationalRefinement_create,
    DISOPTICAL_FLOW_PRESET_ULTRAFAST,
    DISOPTICAL_FLOW_PRESET_FAST,
    DISOPTICAL_FLOW_PRESET_MEDIUM,
    FastOpticalFlowBM,
    calcOpticalFlowBM,
    SparsePyrLKOpticalFlow,
    SparsePyrLKOpticalFlow_create,
    OPTFLOW_USE_INITIAL_FLOW,
    OPTFLOW_FARNEBACK_GAUSSIAN,
)
from ._lib import B2FError  # noqa: F401
from .frames import interpolateFrames  # noqa: F401
from .video import VideoFlow  # noqa: F401
from . import flowio  # noqa: F401
from .superres import (  # noqa: F401
    createSuperResolution_BTVL1_CUDA,
    createOptFlow_Farneback_CUDA,
    createOptFlow_DualTVL1_CUDA,
    createOptFlow_Brox_CUDA,
    createOptFlow_PyrLK_CUDA,
)
from .cudaimgproc import (  # noqa: F401
    CornernessCriteria,
    CornersDetector,
    createHarrisCorner,
    createMinEigenValCorner,
    createGoodFeaturesToTrackDetector,
)
from .lkpyramid import buildOpticalFlowPyramid, calcOpticalFlowPyrLK  # noqa: F401
from . import optflowgf  # noqa: F401
from .optflowgf import calcOpticalFlowFarneback  # noqa: F401
