"""tests/h264_ref.py against tests/golden/h264_ref_digests.json (tests/golden/make_golden_h264_ref.py): every frame of
every clip the CPU video tests code keeps its bytes, macroblock types, Intra 4x4 modes and vectors.  The clips come
from the test modules' cached helpers, so a session that runs those tests too codes each clip once."""
import json
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden_h264_ref import OUT, clips, digest  # noqa: E402

CLIPS = dict(clips())
with open(OUT) as _f:
    WANT = json.load(_f)


def test_digests_cover_every_clip():
    assert sorted(WANT["frames"]) == sorted(CLIPS)


@pytest.mark.parametrize("key", sorted(CLIPS))
def test_clip_keeps_its_digests(key):
    assert [digest(f) for f in CLIPS[key]()] == WANT["frames"][key]
