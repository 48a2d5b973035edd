"""Writes dense_launch_trace.json: every launch, in order and with every argument, that linear_act, mlp_chain,
cross_v2_layer and crossnet_mix_layer issue for the cases and matmul precisions of
tests/test_dense_launch_trace_host.py (which holds the cases and the recorder, and compares against this file).
No GPU and no reference are needed: `_lib.call` is recorded, nothing is launched.

    python tests/golden/make_dense_launch_trace.py

Run it at a commit whose launches are known to be right, and commit the file with the change that means to
alter them; a change that only reorganises the host code must leave the file as it is.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import test_dense_launch_trace_host as T  # noqa: E402

if __name__ == "__main__":
    blob = T.trace_all()
    with open(T.GOLDEN_FILE, "w") as fd:
        fd.write('{"launches": [\n')
        fd.write(",\n".join(json.dumps(rec) for rec in blob["launches"]))
        fd.write('\n],\n"traces": {\n')
        fd.write(",\n".join("%s: %s" % (json.dumps(case), json.dumps(per)) for case, per in blob["traces"].items()))
        fd.write("\n}}\n")
    print("wrote %s: %d distinct launches, %d traces" % (T.GOLDEN_FILE, len(blob["launches"]),
                                                         sum(len(per) for per in blob["traces"].values())))
