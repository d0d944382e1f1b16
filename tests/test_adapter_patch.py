"""The Ceres-side patch of the drop-in must apply to the ceres-solver tree it was generated from, and after it the virtuals
B200Jacobian overrides must no longer be `final` (otherwise the adapter cannot compile as patched).  The tree is not part
of this repository: tools/make_reference_digests.py checked that tools/make_adapter_patch.py regenerates the committed
patch byte for byte from it and that `patch -p1` applies it, and recorded the patch's SHA-256 in
tests/golden/ceres_reference_digests.json.  Here the committed patch must be that patch, and its hunks must do what the
adapter needs."""
import hashlib
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ["internal/ceres/block_sparse_matrix.h", "internal/ceres/evaluator.cc", "internal/ceres/linear_solver.cc",
         "internal/ceres/trust_region_minimizer.cc"]


def _hunks(patch):
    """{file: (removed lines, new side = context + added lines)} of a unified diff."""
    out, cur = {}, None
    for line in patch.splitlines():
        if line.startswith("+++ b/"):
            cur = out.setdefault(line[6:], ([], []))
        elif cur is None or line.startswith(("--- ", "@@", "#")):
            continue
        elif line.startswith("-"):
            cur[0].append(line[1:])
        else:
            cur[1].append(line[1:])
    return out


def test_patch_is_current_and_applies():
    with open(os.path.join(ROOT, "adapter", "ceres_b200.patch"), "rb") as f:
        raw = f.read()
    with open(os.path.join(ROOT, "tests", "golden", "ceres_reference_digests.json")) as f:
        golden = json.load(f)
    assert hashlib.sha256(raw).hexdigest() == golden["patch"], \
        "adapter/ceres_b200.patch is not the patch verified against the ceres-solver tree: regenerate it with " \
        "tools/make_adapter_patch.py and the digests with tools/make_reference_digests.py"
    hunks = _hunks(raw.decode())
    assert sorted(hunks) == sorted(FILES)
    removed, new = hunks[FILES[0]]
    assert "class CERES_NO_EXPORT BlockSparseMatrix : public SparseMatrix {" in new
    # every virtual the adapter overrides is overridable after the patch
    header = open(os.path.join(ROOT, "adapter", "b200_adapter.h")).read()
    jac = header[header.index("class B200Jacobian"):header.index("class B200Evaluator")]
    names = set(re.findall(r"void (\w+)\(", jac)) - {"SyncValuesToHost"}
    assert names == {"SquaredColumnNorm", "ScaleColumns", "RightMultiplyAndAccumulate", "LeftMultiplyAndAccumulate", "SetZero"}
    new_text = "\n".join(new)
    iface = new_text[new_text.index("// Implementation of SparseMatrix interface."):new_text.index("// Convert to CompressedRowSparseMatrix")]
    for n in names:
        decls = re.findall(r"void %s\([^;]*;" % n, iface, flags=re.S)
        assert len(decls) == 2 and all("final" not in d for d in decls), (n, decls)
        assert any(n in r and "final" in r for r in removed), n
    for rel, needle in ((FILES[1], "B200Evaluator::Create(options, program, error)"), (FILES[2], "B200IterativeSchurSolver"),
                        (FILES[3], "ModelCostChange")):
        assert needle in "\n".join(hunks[rel][1])
