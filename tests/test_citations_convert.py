"""The `file:line` citations of the reference in the conversion oracle (oracle_convert/) resolve as test_citations.py requires of the
ABI header, the docs, oracle/ and the CUDA sources: an existing file of the reference tree with at least that many lines."""
import json
import os

from tests.test_citations import GOLDEN, PAT, ROOT


def test_conversion_oracle_citations_resolve():
    with open(GOLDEN) as fh:
        counts = json.load(fh)
    files = {}
    for rel in counts:
        files.setdefault(os.path.basename(rel), []).append(rel)
    d = os.path.join(ROOT, "oracle_convert")
    checked, bad = 0, []
    for f in sorted(os.listdir(d)):
        if not f.endswith((".h", ".cpp", ".py")):
            continue
        for m in PAT.finditer(open(os.path.join(d, f), errors="ignore").read()):
            path, last = m.group(1), int(m.group(3) or m.group(2))
            base = os.path.basename(path)
            if base.startswith(("fls_", "orc_")):
                continue  # this repository's own files
            checked += 1
            cands = files.get(base, [])
            if "/" in path:
                cands = [c for c in cands if ("/" + c).endswith("/" + path.lstrip("./"))] or cands
            if not cands:
                bad.append((f, m.group(0), "no such file in the reference"))
            elif max(counts[c] for c in cands) < last:
                bad.append((f, m.group(0), "file is shorter than the cited line"))
    assert checked > 0
    assert not bad, bad
