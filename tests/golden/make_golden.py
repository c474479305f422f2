"""Generates tests/golden/* from the reference's OWN artefacts, so that the tests need no copy of the reference.  Run:
    python tests/golden/make_golden.py <shifu-tensorflow checkout>/shifu-tensorflow-eval/src/test/resources/dummydl

dummydl_known_answers.json : forward outputs of the reference's SavedModel fixture
    (shifu-tensorflow-eval/src/test/resources/dummydl, loaded by TensorflowModelTest.java:35-60) computed by the
    oracle reader + fp32 numpy forward.  NOT TF-verified (TF is not installable here); they agree with the values
    SURVEY.md section 8c lists, which were derived independently.
dummydl_op_attrs.json : for every op type in the fixture's GraphDef (written by a real TF 1.x), the attribute keys its
    nodes carry, plus the attribute keys of the SignatureDef / SaverDef plumbing - the structural reference our own
    SavedModel writer is linted against (tests/test_formats.py).
dummydl_head.npz : the first 3 and the last layer of that model + a 16-row input/output pair, small enough to
    commit, so the scorer kernels can be checked against the fixture's real weights.
dummydl_saved_model.pb.xz, dummydl_variables.index : the fixture's GraphDef and tensor-bundle index exactly as TF wrote
    them (xz-compressed graph).  With the stored tensors written at the index's offsets into a (sparse) data file they make
    the fixture again: tests/test_formats.py rebuilds it so that both readers run on a TF-written model.
dummydl_mlp_mid.npz : layers 3..19 of the MLP as the oracle reader extracts it (dummydl_head.npz holds the others), with
    the variable names and activations of all 21 layers; checked against the index's crcs.
"""
import json
import lzma
import os
import shutil
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import tf_formats as tff  # noqa: E402



def main(fixture):
    FIXTURE = fixture
    layers, names = tff.extract_mlp(FIXTURE, "dense_46_input", "dense_66/Sigmoid")
    cases = []
    for value in (0.5, 0.0):
        X = np.full((1, 1522), value, np.float32)
        cases.append({"input_fn": "const", "value": value, "expected": [float(v) for v in tff.mlp_forward(layers, X).ravel()]})
    X = np.random.RandomState(0).rand(4, 1522).astype(np.float32)
    cases.append({"input_fn": "rand", "seed": 0, "rows": 4, "expected": [float(v) for v in tff.mlp_forward(layers, X).ravel()]})
    json.dump({"source": "dummydl fixture via oracle/tf_formats.py", "input": "dense_46_input", "output": "dense_66/Sigmoid",
               "cases": cases}, open(os.path.join(HERE, "dummydl_known_answers.json"), "w"), indent=1)
    # reduced model: layers 0,1,2 + output layer (1522->100->100->100->1), fp16-free, ~650 KB compressed
    sub = [layers[0], layers[1], layers[2], layers[-1]]
    X = np.random.RandomState(1).rand(16, 1522).astype(np.float32)
    Y = tff.mlp_forward(sub, X)
    np.savez_compressed(os.path.join(HERE, "dummydl_head.npz"), X=X, Y=Y,
                        **{"W%d" % i: l[0] for i, l in enumerate(sub)}, **{"b%d" % i: l[1] for i, l in enumerate(sub)})
    nodes, sigs = tff.read_graph_nodes(os.path.join(FIXTURE, "saved_model.pb"))
    ops = {}
    for _name, (op, _inputs, attrs) in nodes.items():
        ops.setdefault(op, set()).update(attrs.keys())
    json.dump({"source": "dummydl/saved_model.pb (TF-written GraphDef), via oracle/tf_formats.read_graph_nodes",
               "op_attr_keys": {op: sorted(keys) for op, keys in sorted(ops.items())}, "signatures": sorted(sigs)},
              open(os.path.join(HERE, "dummydl_op_attrs.json"), "w"), indent=1)
    shutil.copyfile(os.path.join(FIXTURE, "variables", "variables.index"), os.path.join(HERE, "dummydl_variables.index"))
    with open(os.path.join(FIXTURE, "saved_model.pb"), "rb") as f, lzma.open(os.path.join(HERE, "dummydl_saved_model.pb.xz"), "wb",
                                                                          preset=9 | lzma.PRESET_EXTREME) as g:
        g.write(f.read())
    mid = {i: l for i, l in enumerate(layers) if 3 <= i < len(layers) - 1}
    np.savez_compressed(os.path.join(HERE, "dummydl_mlp_mid.npz"), acts=np.array([l[2] for l in layers], np.int32),
                        names=np.array([n for pair in names for n in pair]),
                        **{"W%d" % i: l[0] for i, l in mid.items()}, **{"b%d" % i: l[1] for i, l in mid.items()})
    print("wrote", os.listdir(HERE))


if __name__ == "__main__":
    main(sys.argv[1])
