"""Every `file:line` citation of the reference in the ABI header, the docs, the oracle and the CUDA sources must point at
an existing file of the reference tree with at least that many lines.  The reference tree is described by
tests/golden/reference_line_counts.json (path relative to the reference root -> number of lines), regenerated with
`python tests/golden/make_golden.py --reference-tree DIR`."""
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_line_counts.json")
PAT = re.compile(r"([A-Za-z0-9_/\.]+\.(?:h|cpp|yaml|md|txt)):(\d+)(?:-(\d+))?")


def _sources():
    out = [os.path.join(ROOT, p) for p in ("DESIGN.md", "INTEGRATION.md", "include/fls_b200.h", "funny_lidar_slam_b200/shim/b200_registration.h")]
    for d, exts in (("oracle", (".h", ".cpp", ".py")), ("funny_lidar_slam_b200/csrc", (".cu", ".cuh", ".h"))):
        out += [os.path.join(ROOT, d, f) for f in sorted(os.listdir(os.path.join(ROOT, d))) if f.endswith(exts)]
    return out


def test_reference_citations_resolve():
    with open(GOLDEN) as fh:
        counts = json.load(fh)
    files = {}
    for rel in counts:
        files.setdefault(os.path.basename(rel), []).append(rel)

    checked, bad = 0, []
    for src in _sources():
        for m in PAT.finditer(open(src, errors="ignore").read()):
            path, last = m.group(1), int(m.group(3) or m.group(2))
            base = os.path.basename(path)
            if base.startswith(("fls_", "orc_")) or base == "b200_registration.h":
                continue  # this repository's own files
            checked += 1
            cands = files.get(base, [])
            if "/" in path:
                cands = [c for c in cands if ("/" + c).endswith("/" + path.lstrip("./"))] or cands
            if not cands:
                bad.append((os.path.relpath(src, ROOT), m.group(0), "no such file in the reference"))
            elif max(counts[c] for c in cands) < last:
                bad.append((os.path.relpath(src, ROOT), m.group(0), "file is shorter than the cited line"))
    assert checked > 150
    assert not bad, bad
