"""Writes tests/golden/jpeg/digests.json: SHA-256 of the CPU decoder's RGB output (torchvision.io.decode_jpeg,
mode=RGB, libjpeg-turbo) for the two camera files and the seeded 61x117 part of the corpus, each beside the digest of
the file it decoded.  The tests compare against these, so the decoder the device path reproduces stays pinned even
where another torchvision (or PIL, for the generated files) is installed.

    python oracle/make_golden_jpeg.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import jpeg_corpus as J  # noqa: E402


def main():
    files = J.assets() + [(n, b) for n, b, _ in J.corpus(sizes=((61, 117),))]
    out = {name: {"file": J.sha(data), "rgb": J.sha(J.cpu_decode(data).numpy().tobytes())} for name, data in files}
    path = os.path.join(J.GOLDEN_JPEG, "digests.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path, len(out), "digests")


if __name__ == "__main__":
    main()
