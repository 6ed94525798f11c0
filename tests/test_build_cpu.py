"""The library build's dependency list: an edit to any header a translation unit includes must rebuild the units, so
every header under csrc/ and every header a csrc file includes is in `build.headers()`."""
import glob
import os
import re

from cudasift_b200 import build


def test_every_csrc_header_is_a_dependency():
    deps = set(map(os.path.realpath, build.headers()))
    found = glob.glob(os.path.join(build.CSRC, "*.cuh")) + glob.glob(os.path.join(build.CSRC, "*.h"))
    assert any(f.endswith("sift_arith.cuh") for f in found)
    missing = sorted(os.path.basename(f) for f in found if os.path.realpath(f) not in deps)
    assert not missing, "headers under csrc/ that do not trigger a rebuild: %s" % missing


def test_every_included_header_is_a_dependency():
    deps = set(map(os.path.realpath, build.headers()))
    missing = []
    for src in sorted(glob.glob(os.path.join(build.CSRC, "*"))):
        if not src.endswith((".cu", ".cuh", ".h")):
            continue
        with open(src) as f:
            for name in re.findall(r'^\s*#\s*include\s+"([^"]+)"', f.read(), re.M):
                path = os.path.realpath(os.path.join(os.path.dirname(src), name))
                if path not in deps:
                    missing.append("%s: %s" % (os.path.basename(src), name))
    assert not missing, "included headers that do not trigger a rebuild: %s" % missing
