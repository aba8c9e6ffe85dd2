#!/usr/bin/env python
"""Extract the reference's own known-answer tests for the hot path into JSON.

TensorFlow cannot be imported in the build image, so instead of *running* the
reference this script parses the reference's test files with `ast` and lifts
the literal inputs and expected outputs out of them (evaluating only numpy
expressions; `tf.constant` / `tf.ragged.constant` are stubbed to numpy/lists).
Run it against a checkout of the reference; the JSON it writes is committed, so
the tests never need the reference itself.

    python tests/golden/extract_reference_kats.py <path to the reference checkout>

Output: tests/golden/reference_kats.json
"""
import ast
import json
import os
import sys
import types

import numpy as np

if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
TESTS = os.path.join(REF, "tests", "ampligraph", "latent_features")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_kats.json")

_tf = types.SimpleNamespace(
    constant=lambda x, dtype=None: np.array(x, dtype=np.float32 if dtype == "f32" else None),
    float32="f32", int32="i32",
    ragged=types.SimpleNamespace(constant=lambda x, dtype=None: x),
)
_ENV = {"np": np, "tf": _tf}


def _ev(node, extra=None):
    env = dict(_ENV)
    if extra:
        env.update(extra)
    return eval(compile(ast.Expression(node), "<kat>", "eval"), env)


def _lst(a):
    return np.asarray(a).tolist()


def _funcs(path):
    with open(path) as f:
        tree = ast.parse(f.read())
    return {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef)}, path


def _assigns(fn):
    """name -> value node for simple `name = expr` statements, in order."""
    out = []
    for st in fn.body:
        if isinstance(st, ast.Assign) and len(st.targets) == 1 and isinstance(st.targets[0], ast.Name):
            out.append((st.targets[0].id, st.value, st.lineno))
    return out


def _compare_rhs(node):
    """right-hand side of the first `lhs == rhs` comparison under node (e.g.
    `2 * np.array([...]) / 3.0` in test_HolE.py)."""
    for n in ast.walk(node):
        if isinstance(n, ast.Compare) and isinstance(n.ops[0], ast.Eq):
            return n.comparators[0]
    return None


def _first_np_array_in(node):
    for n in ast.walk(node):
        if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == "array" \
                and isinstance(n.func.value, ast.Name) and n.func.value.id == "np":
            return n
    return None


def scoring_kats():
    out = []
    for name in ("TransE", "DistMult", "ComplEx", "HolE", "RotatE"):
        rel = os.path.join("layers", "scoring", "test_%s.py" % name)
        funcs, path = _funcs(os.path.join(TESTS, rel))
        for fname, form in (("test_compute_score", "triple"),
                            ("test_get_subject_corruption_scores", "sub_diag"),
                            ("test_get_object_corruption_scores", "obj_diag")):
            fn = funcs[fname]
            vals, ctor = {}, None
            for nm, node, _ in _assigns(fn):
                if nm in ("triples", "ent_matrix"):
                    vals[nm] = _ev(node)
                if nm == "model":
                    ctor = {kw.arg: _ev(kw.value) for kw in node.keywords}
            expected = None
            for st in fn.body:
                if isinstance(st, ast.Assert):
                    expected = _ev(_compare_rhs(st.test))
            out.append({
                "source": "tests/ampligraph/latent_features/%s::%s:%d" % (rel, fname, fn.lineno),
                "model": name, "form": form, "k": ctor["k"],
                "max_rel_size": ctor.get("max_rel_size"),
                "e_s": _lst(vals["triples"][0]), "e_p": _lst(vals["triples"][1]),
                "e_o": _lst(vals["triples"][2]),
                "ent_matrix": _lst(vals["ent_matrix"]) if "ent_matrix" in vals else None,
                "round_decimals": 2, "expected": _lst(expected),
            })
    return out


def rank_kats():
    rel = os.path.join("layers", "scoring", "test_AbstractScoringLayer.py")
    funcs, _ = _funcs(os.path.join(TESTS, rel))
    fn = funcs["test_compute_score"]
    vals, cases, pending = {}, [], None
    for st in fn.body:
        if isinstance(st, ast.Assign) and isinstance(st.targets[0], ast.Name):
            nm = st.targets[0].id
            if nm in ("triples", "ent_matrix"):
                vals[nm] = _ev(st.value)
            elif nm == "model":
                vals["k"] = _ev(st.value.keywords[0].value)
                vals["model"] = st.value.func.id
            elif nm == "ranks":
                call = st.value
                args = call.args
                pending = {
                    "start_ent_id": _ev(args[2]), "end_ent_id": _ev(args[3]),
                    "filters": _ev(args[4]),
                    "corrupt_side": "s,o", "comparison_type": "worst", "line": st.lineno,
                }
                for kw in call.keywords:
                    pending[kw.arg] = _ev(kw.value)
        elif isinstance(st, ast.Assert) and pending is not None:
            pending["expected"] = _lst(_ev(_first_np_array_in(st.test)))
            cases.append(pending)
            pending = None
    return {
        "source": "tests/ampligraph/latent_features/%s::test_compute_score:%d" % (rel, fn.lineno),
        "model": vals["model"], "k": vals["k"],
        "e_s": _lst(vals["triples"][0]), "e_p": _lst(vals["triples"][1]), "e_o": _lst(vals["triples"][2]),
        "ent_matrix": _lst(vals["ent_matrix"]), "cases": cases,
        "note": "expected values are the counts returned by get_ranks, i.e. BEFORE evaluate() adds 1",
    }


_LOSS_NAMES = {"PairwiseLoss": "pairwise", "NLLLoss": "nll", "AbsoluteMarginLoss": "absolute_margin",
               "SelfAdversarialLoss": "self_adversarial", "NLLMulticlass": "multiclass_nll"}


def loss_kats():
    rel = "test_loss_functions.py"
    funcs, _ = _funcs(os.path.join(TESTS, rel))
    out = []
    for fname, fn in funcs.items():
        cls_name = fname[len("test_"):]
        if cls_name not in _LOSS_NAMES:
            continue
        cur = {}
        for st in fn.body:
            if isinstance(st, ast.Assign) and isinstance(st.targets[0], ast.Name):
                nm = st.targets[0].id
                if nm == "lossObj":
                    cur = {"params": _ev(st.value.args[0]) if st.value.args else {}}
                elif nm in ("pos_score", "corr_score"):
                    cur[nm] = _lst(np.asarray(_ev(st.value), dtype=np.float32))
                elif nm == "loss":
                    cur["eta"] = [_ev(kw.value) for kw in st.value.keywords if kw.arg == "eta"][0]
                    cur["line"] = st.lineno
            elif isinstance(st, ast.Assert) and "eta" in cur and "expected_per_positive" not in cur:
                arr = _first_np_array_in(st.test)
                if arr is None:
                    continue
                cur["expected_per_positive"] = _lst(_ev(arr))
                out.append({
                    "source": "tests/ampligraph/latent_features/%s::%s:%d" % (rel, fname, cur["line"]),
                    "loss": _LOSS_NAMES[cls_name], "params": cur["params"], "eta": cur["eta"],
                    "pos_score": cur["pos_score"], "corr_score": cur["corr_score"],
                    "expected_per_positive": cur["expected_per_positive"], "tol": 1e-4,
                    "note": "the reference asserts sum(expected_per_positive) against the scalar loss",
                })
    return out


def lookup_kat():
    rel = os.path.join("layers", "encoding", "test_EmbeddingLookupLayer.py")
    funcs, _ = _funcs(os.path.join(TESTS, rel))
    fn = funcs["test_call"]
    inits, sample, expected = None, None, []
    for n in ast.walk(fn):
        if isinstance(n, ast.keyword) and n.arg == "entity_relation_initializer":
            inits = [_ev(c.args[0]) for c in n.value.elts]
        if isinstance(n, ast.keyword) and n.arg == "sample":
            sample = _ev(n.value.args[0])
    for st in fn.body:
        if isinstance(st, ast.Assert):
            expected.append(_lst(_ev(_first_np_array_in(st.test))))
    return {"source": "tests/ampligraph/latent_features/%s::test_call:%d" % (rel, fn.lineno),
            "ent_emb": inits[0], "rel_emb": inits[1], "sample": sample,
            "expected_s_p_o": expected}


def corruption_kat():
    rel = os.path.join("layers", "corruption_generation", "test_CorruptionGenerationLayerTrain.py")
    funcs, _ = _funcs(os.path.join(TESTS, rel))
    fn = funcs["test_call"]
    pos = ent_size = eta = expected = None
    for n in ast.walk(fn):
        if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == "call":
            pos, ent_size, eta = _lst(_ev(n.args[0])), _ev(n.args[1]), _ev(n.args[2])
    for st in fn.body:
        if isinstance(st, ast.Assert):
            expected = _lst(_ev(_first_np_array_in(st.test)))
    return {"source": "tests/ampligraph/latent_features/%s::test_call:%d" % (rel, fn.lineno),
            "pos": pos, "ent_size": ent_size, "eta": eta, "expected_with_tf_seed_0": expected,
            "note": "ids depend on TensorFlow's stateful RNG stream (tf.random.set_seed(0)); only the "
                    "STRUCTURE is reproducible: tile order, exactly one side replaced, relation kept, "
                    "ids < ent_size"}


def main():
    kats = {
        "generated_by": "tests/golden/extract_reference_kats.py",
        "reference": "Accenture/AmpliGraph @ 260a732",
        "scoring": scoring_kats(),
        "ranks": rank_kats(),
        "losses": loss_kats(),
        "lookup": lookup_kat(),
        "corruption": corruption_kat(),
    }
    with open(OUT, "w") as f:
        json.dump(kats, f, indent=1, sort_keys=True)
    print("wrote %s: %d scoring, %d rank cases, %d loss KATs" % (
        OUT, len(kats["scoring"]), len(kats["ranks"]["cases"]), len(kats["losses"])))


if __name__ == "__main__":
    main()
