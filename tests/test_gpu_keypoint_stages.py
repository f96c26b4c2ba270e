"""`-m gpu`: the face / hand crop pass of opb_keypoints_detect_crops run stage by stage on the H100 from injected maps
(opb_test_keypoint_stages, tests/keypoint_stages.py) at a network size of 368: every canvas byte, upsampled, axis-0
and smoothed float, arg-max record and keypoint of seven crop tables (1 to 301 crops, 70 and 21 planes, three frames)
bit for bit against cv2, scipy and the restated reference, with sentinels past every buffer."""
import pytest

import keypoint_stages as K
from conftest import pkg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    return pkg("_native").Engine(0, pkg("pose_detector").make_opb_params())


def test_keypoint_stages(engine):
    stats = K.run_all(engine)
    print("keypoint stages: %s" % stats)


def test_keypoint_stages_argument_errors(engine):
    K.check_argument_errors(engine)
