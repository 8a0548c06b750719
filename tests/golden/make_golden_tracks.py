"""Records tests/golden/reference_tracks.json: runs the reference's unmodified lib/tracks.py (path given as the first argument,
`aiortc` stubbed) with the fake source and recording pipeline of tests/test_tracks.py, and stores the frames it returned, the
pipeline calls it made and its warm-up counter for DROP_FRAMES = 0 and 1.

    python tests/golden/make_golden_tracks.py <reference checkout>/lib/tracks.py
"""
import importlib.util
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import test_tracks as T  # noqa: E402


def main(path):
    aiortc = types.ModuleType("aiortc")

    class MediaStreamTrack:
        def __init__(self):
            self._ended = False

    aiortc.MediaStreamTrack = MediaStreamTrack
    sys.modules["aiortc"] = aiortc
    out = {}
    for drop in (0, 1):
        os.environ.pop("WARMUP_FRAMES", None)
        os.environ["DROP_FRAMES"] = str(drop)
        spec = importlib.util.spec_from_file_location("reference_lib_tracks", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        pipe = T.RecordingPipeline()
        track = mod.VideoStreamTrack(T.FakeSource(), pipe)
        res = T._drive(track, 5)
        out[str(drop)] = {"outputs": [list(r) for r in res], "calls": [list(c) for c in pipe.calls],
                          "warmup_frame_idx": track.warmup_frame_idx}
    with open(T.GOLDEN, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
