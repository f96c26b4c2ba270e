"""H100-native OpenPose inference hot path behind the API of the reference's pose_detector.py.

    from <package> import PoseDetector, draw_person_pose, draw_whole_body, detect_whole_body, params, JointType
    from <package> import detect_whole_body_batch
    from <package> import FaceDetector, CascadeClassifier

or, flat like the reference: put this directory on sys.path and `import pose_detector`.
The CUDA library (libopb.so) is built by `__graft_entry__.build()`; importing this package
does not need a GPU, constructing a PoseDetector does."""
from .entity import JointType, params  # noqa: F401
from .pose_detector import PoseDetector, draw_person_pose, make_opb_params  # noqa: F401
from .whole_body import detect_whole_body, detect_whole_body_batch, draw_whole_body  # noqa: F401
from .face_detector import FaceDetector  # noqa: F401
from .cascade import CascadeClassifier  # noqa: F401
from . import _native, synthetic  # noqa: F401
