"""Compile the spatial-tendon test models into tests/golden/{tendon_paths,arm26,newton_cradle}.mjb with the reference's
own compiler and mj_saveModel (the product has no MJCF compiler): models/tendon_paths.xml (authored here) and the
reference's model/tendon_arm/arm26.xml and model/replicate/newton_cradle.xml.  The reference models are compiled as
they are except that their builtin textures are made 8 x 8 pixels: textures only reach rendering, and at 512 x 512
they would make up nearly all of the stored files.  Run where the oracle is built and the reference tree is at
$MJB_REFERENCE.

Usage: python tests/golden/make_tendon_fixtures.py
"""
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_util import Oracle  # noqa: E402

REF = os.environ.get("MJB_REFERENCE", "/root/reference")


def main():
    sources = {"tendon_paths": os.path.join(ROOT, "models", "tendon_paths.xml"),
               "arm26": os.path.join(REF, "model", "tendon_arm", "arm26.xml"),
               "newton_cradle": os.path.join(REF, "model", "replicate", "newton_cradle.xml")}
    for name, src in sources.items():
        with open(src) as f:
            xml = re.sub(r'(<texture[^>]*?)width="\d+" height="\d+"', r'\1width="8" height="8"', f.read())
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, name + ".xml")
            with open(path, "w") as f:
                f.write(xml)
            Oracle(path).save_mjb(os.path.join(ROOT, "tests", "golden", name + ".mjb"))
        print("wrote tests/golden/%s.mjb" % name)


if __name__ == "__main__":
    main()
