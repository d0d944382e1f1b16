"""Records what the adapter tests compare against in a ceres-solver tree, as digests only (no Ceres source is stored):
    python tools/make_reference_digests.py <ceres-solver tree> > tests/golden/ceres_reference_digests.json
  * signatures: SHA-256 of every normalised declaration of tests/test_adapter_mock.py's SIGNATURES that the tree's
    header contains (the script fails if one is missing);
  * patch: SHA-256 of adapter/ceres_b200.patch, after checking that tools/make_adapter_patch.py regenerates it byte
    for byte from the tree and that `patch -p1` applies it there."""
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.test_adapter_mock import SIGNATURES, _norm  # noqa: E402
from tests.test_adapter_patch import FILES  # noqa: E402


def sha(b):
    return hashlib.sha256(b if isinstance(b, bytes) else b.encode()).hexdigest()


ref = sys.argv[1]
sigs = {}
for rel, lst in sorted(SIGNATURES.items()):
    text = _norm(open(os.path.join(ref, rel)).read())
    for s in lst:
        assert _norm(s) in text, (rel, s)
    sigs[rel] = sorted(sha(_norm(s)) for s in lst)
patch_path = os.path.join(ROOT, "adapter", "ceres_b200.patch")
patch = open(patch_path, "rb").read()
gen = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_adapter_patch.py"), ref], capture_output=True, check=True)
assert gen.stdout == patch, "adapter/ceres_b200.patch is stale: regenerate with tools/make_adapter_patch.py"
with tempfile.TemporaryDirectory() as tmp:
    for rel in FILES:
        os.makedirs(os.path.dirname(os.path.join(tmp, rel)), exist_ok=True)
        shutil.copy(os.path.join(ref, rel), os.path.join(tmp, rel))
    subprocess.run(["patch", "-p1", "-i", patch_path], cwd=tmp, check=True, capture_output=True)
json.dump({"patch": sha(patch), "signatures": sigs}, sys.stdout, indent=1, sort_keys=True)
sys.stdout.write("\n")
