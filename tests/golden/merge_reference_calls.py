"""Folds the JSON lines written by tests run with BROTLI_REF_RECORD=<file> (brotli_libs.RecordedRef, oracle/_ref built)
into tests/golden/reference_calls.json, the reference results the tests replay:

    BROTLI_REF_RECORD=/tmp/calls.jsonl python -m pytest tests -m "not gpu" -k "<tests that compare with the reference>"
    python tests/golden/merge_reference_calls.py /tmp/calls.jsonl [...]

A key recorded twice must carry the same value both times (the reference is deterministic for these calls)."""
import json
import os
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_calls.json")

calls = json.load(open(OUT)) if os.path.exists(OUT) else {}
for path in sys.argv[1:]:
    for line in open(path):
        r = json.loads(line)
        v = r["value"] if isinstance(r["value"], int) else [r["value"][0], r["value"][1][:32]]
        old = calls.setdefault(r["key"], v)
        assert old == v, ("the reference gave two results for one call", r["key"])
with open(OUT, "w") as f:       # one call per line
    f.write("{\n" + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(calls[k])) for k in sorted(calls)) + "\n}\n")
print("%d calls in %s" % (len(calls), OUT))
