"""Records tests/golden/functor_edges_reference.json: for every functor edge case of tests/test_functor_edges.py
(cpu_cases, restricted to the rows C++ defines), the digest of the reference's HOST build's outputs (UnaryTransform /
BinaryTransform into every sink, BinaryFilter), with the rows whose conversion into the sink is undefined zeroed.
Needs oracle/_ref (oracle/build_ref.sh over a checkout of the reference)."""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))

import harness as H  # noqa: E402
import test_functor_edges as T  # noqa: E402

assert H.reference_built(), "oracle/_ref is not built"
out = T.reference_digests(H.get_backend("ref"))
T.FIXTURE.write_text(json.dumps(out, indent=0, sort_keys=True) + "\n")
print(len(out), "cases")
