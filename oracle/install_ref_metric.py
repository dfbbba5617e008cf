"""Install the UNMODIFIED reference metric modules (metric/utils.py, metric/metrics.py, metric/lookup_tables.py) into
oracle/_ref/ next to the modules install_ref.py installs, so that tools/surface_bench.py can time the reference's
calculate_distance on the host CPU.  Called by __graft_entry__.build() after install_ref; same source checkout
(B200SEG_REFERENCE), same byte-for-byte copy; the SHA-256 digests go to oracle/_ref/MANIFEST_metric.json (install_ref
owns MANIFEST.json).  Does nothing when the checkout is absent, keeping whatever oracle/_ref/ already holds."""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from install_ref import DST, REF    # noqa: E402

FILES = ["metric/utils.py", "metric/metrics.py", "metric/lookup_tables.py"]


def main():
    if not os.path.isdir(REF):
        print("install_ref_metric: %s not present — keeping whatever oracle/_ref already holds" % REF)
        return 0
    manifest = {}
    for rel in FILES:
        src = os.path.join(REF, rel)
        if not os.path.exists(src):
            continue
        dst = os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        manifest[rel] = hashlib.sha256(open(dst, "rb").read()).hexdigest()
    json.dump({"source": REF, "sha256": manifest}, open(os.path.join(DST, "MANIFEST_metric.json"), "w"), indent=1)
    print("install_ref_metric: %d reference files -> %s" % (len(manifest), DST))
    return 0


if __name__ == "__main__":
    sys.exit(main())
