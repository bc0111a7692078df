"""Write the digests of the stored LDL^T factor on the matrices of tests/factor_digest.py (needs a GPU).
Usage: python scripts/make_factor_digests.py OUT.json   (tests/golden/ldl/factor_digests.json is the committed copy)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import factor_digest  # noqa: E402

out = {}
for case in factor_digest.cases():
    s = factor_digest.solver(case)
    out[case.name] = factor_digest.digest(s)
    s.close()
    print(case.name, out[case.name])
with open(sys.argv[1], "w") as fp:
    json.dump(out, fp, indent=1, sort_keys=True)
    fp.write("\n")
