"""Generate tests/golden/h264_ref_digests.json: SHA-256 digests of every frame tests/h264_ref.py codes for the CPU
video tests, so that a change to the restatement that moves a byte, a macroblock type, an Intra 4x4 mode or a vector
fails tests/test_h264_ref.py.

    python tests/golden/make_golden_h264_ref.py

"frames": per clip, each frame's digests of its bytes and of its types, modes and mv arrays.  The clips are the
gop_cases, me_cases and i4_cases of tests/test_video_{gop,me,i4}.py at each of their GOPS, the 52-qp sweep of
test_video_gop.py and the noise clips of the three bound tests, each coded as its test codes it.
"zero_motion": the digests of the bytes of the me_cases at search 0, gop 2 and T.
"without_i4": the digests of the bytes of the i4_cases without Intra 4x4, at their search, gop 2 and T.
The digests were first made by the three restatements this module's one replaced (the zero-motion GOP rule, the
motion search rule and the Intra 4x4 rule), each clip by the one that coded it, so the last two sections hold the
bytes of the zero-motion and motion search restatements: tests/test_video_me.py and tests/test_video_i4.py compare
search 0 and the rule without Intra 4x4 with them."""
import functools
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
OUT = os.path.join(HERE, "h264_ref_digests.json")


def _sha(b):
    return hashlib.sha256(b).hexdigest()


def _array(a):
    """The digest of an int array or of an array of macroblock type strings, with its shape."""
    a = np.asarray(a, "U4" if a.dtype == object else np.int64)
    return _sha(repr(a.shape).encode() + a.tobytes())


def digest(frame):
    return {"data": _sha(frame.data), "types": _array(frame.types), "modes": _array(frame.modes),
            "mv": None if frame.mv is None else _array(frame.mv)}


def clips():
    """(key, encode) of every clip of "frames": encode() returns its frames from the test module's cached helper."""
    import test_video_gop as tg
    import test_video_i4 as ti
    import test_video_me as tm
    out = [(f"{tag}/{c[0]}/{g}", functools.partial(mod.encoded, c[0], g))
           for tag, mod, cases in (("gop", tg, tg.gop_cases()), ("me", tm, tm.me_cases()), ("i4", ti, ti.i4_cases()))
           for c in cases for g in mod.GOPS]
    out += [(f"gop/every_qp/{qp}", functools.partial(tg.every_qp, qp)) for qp in range(52)]
    out += [(f"gop/noise/{qp}", functools.partial(tg.noise_bound, qp)) for qp in (0, 51)]
    out += [("me/noise", tm.noise_bound)]
    out += [(f"i4/noise/{gop}", functools.partial(ti.noise_bound, gop)) for gop in (1, 3)]
    return out


def baselines():
    """(section, key, frames, qp, gop, search) of the "zero_motion" and "without_i4" clips."""
    import test_video_i4 as ti
    import test_video_me as tm
    for name, frames, qp, _, _ in tm.me_cases():
        for gop in (2, len(frames)):
            yield "zero_motion", f"{name}/{gop}", frames, qp, gop, 0
    for name, frames, qp, search in ti.i4_cases():
        for gop in (2, len(frames)):
            yield "without_i4", f"{name}/{gop}", frames, qp, gop, search


def main():
    sys.path[:0] = [ROOT, TESTS]
    import h264_ref
    out = {"frames": {key: [digest(f) for f in encode()] for key, encode in clips()},
           "zero_motion": {}, "without_i4": {}}
    for section, key, frames, qp, gop, search in baselines():
        out[section][key] = [_sha(f.data) for f in h264_ref.encode_clip(frames, qp, gop, search)]
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
