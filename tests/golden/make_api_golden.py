"""Golden outputs of UNMODIFIED reference code for tests/test_api.py, written to tests/golden/api_reference.json.

Run from the repository root with a checkout of the reference DensePhrases repository:
    python tests/golden/make_api_golden.py /path/to/DensePhrases
It executes, over this repository's drop-in surface (the same inputs the tests use):
  - the `densephrases.*` imports of eval_phrase_retrieval.py (:12-25), recorded as (module, names);
  - eval_phrase_retrieval.evaluate (:49-91) + evaluate_results (:94-204) with canned encoder / MIPS stand-ins;
  - DensePhrases.search of densephrases/model.py:55-109 over this repo's MIPS / query2vec, for every retrieval unit;
  - load_qa_pairs (open_utils.py:103-163) and backward_compat (single_utils.py:36-56);
  - the Options parser (options.py) defaults and one argv;
  - TrueCaser (squad_utils.py:1452-1585) on seeded random sentences."""
import ast
import importlib.util
import json
import math
import os
import pickle
import string
import sys
import tempfile
import types
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import test_api as T  # noqa: E402  (inputs shared with the tests)


def load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def with_stubs(stubs, fn):
    for name, attrs in stubs.items():
        m = types.ModuleType(name)
        for a in attrs:
            setattr(m, a, type(a, (), {}) if a == "TrueCaser" else object)
        sys.modules[name] = m
    try:
        return fn()
    finally:
        for name in stubs:
            del sys.modules[name]


def imports_of(path):
    out = []
    for node in ast.parse(open(path).read()).body:
        if isinstance(node, ast.ImportFrom) and node.module and node.module.startswith("densephrases"):
            out.append([node.module, [a.name for a in node.names]])
        elif isinstance(node, ast.Import):
            out.extend([[a.name, []] for a in node.names if a.name in ("faiss",) or a.name.startswith("densephrases")])
    return out


def main(ref):
    import numpy as np
    from oracle import ivfpq_ref
    ivfpq_ref.build()
    g = {"imports": imports_of(os.path.join(ref, "eval_phrase_retrieval.py"))}

    # eval_phrase_retrieval.evaluate
    mod = load("ref_eval_phrase_retrieval_run", os.path.join(ref, "eval_phrase_retrieval.py"))
    with tempfile.TemporaryDirectory() as tmp:
        args, mips, enc, tok = T.reference_evaluate_inputs(tmp)
        em1, f11, emk, f1k = mod.evaluate(args, mips=mips, query_encoder=enc, tokenizer=tok)
        g["evaluate"] = {"em1": em1, "f1_1": f11, "emk": emk, "f1_k": f1k, "pred": json.load(open(os.path.join(tmp, "pred", "test_5_top3.pred")))}

    # DensePhrases.search (model.py)
    model = with_stubs({"densephrases.utils.squad_utils": ("TrueCaser",)}, lambda: load("ref_densephrases_model", os.path.join(ref, "densephrases", "model.py")))
    g["search"] = {}
    for unit in ("phrase", "sentence", "paragraph", "document"):
        theirs = model.DensePhrases.__new__(model.DensePhrases)
        qs = T.search_wrapper_setup(ivfpq_ref, theirs)
        a = theirs.search(qs, retrieval_unit=unit, top_k=3, truecase=False, return_meta=True)
        g["search"][unit] = {"results": a[0], "meta": T.strip_vectors(a[1]),
                             "single": theirs.search(qs[0], retrieval_unit=unit, top_k=2, truecase=False)}

    # load_qa_pairs / backward_compat
    stubs = {"densephrases.utils.squad_utils": ("get_question_dataloader", "TrueCaser"), "densephrases.utils.embed_utils": ("get_question_results",)}
    mods = with_stubs(stubs, lambda: {s: load(f"ref_{s}", os.path.join(ref, "densephrases", "utils", f"{s}.py")) for s in ("single_utils", "open_utils")})
    with tempfile.TemporaryDirectory() as tmp:
        p = T.write_qa_pairs_input(tmp)
        g["load_qa_pairs"] = []
        for lower, q_idx in T.QA_PAIR_CASES:
            T.QaArgs.do_lower_case = lower
            g["load_qa_pairs"].append([list(x) for x in mods["open_utils"].load_qa_pairs(p, T.QaArgs, q_idx=q_idx)])
    g["backward_compat"] = mods["single_utils"].backward_compat(dict(T.BACKWARD_COMPAT_SD))

    # Options
    opts = load("ref_options", os.path.join(ref, "densephrases", "options.py"))
    theirs = opts.Options()
    for group in ("add_model_options", "add_index_options", "add_retrieval_options", "add_data_options"):
        getattr(theirs, group)()
    g["options_defaults"] = vars(theirs.parser.parse_args([]))
    g["options_argv"] = vars(theirs.parser.parse_args(T.OPTIONS_ARGV))

    # TrueCaser
    def cut(path, name):
        src = open(path).read()
        node = next(n for n in ast.parse(src).body if getattr(n, "name", None) == name)
        return ast.get_source_segment(src, node)
    ns = {"os": os, "pickle": pickle, "math": math, "string": string}
    exec(cut(os.path.join(ref, "densephrases", "utils", "data_utils.py"), "whitespace_tokenize"), ns)
    exec(cut(os.path.join(ref, "densephrases", "utils", "squad_utils.py"), "TrueCaser"), ns)
    tables = pickle.load(open(T.TRUECASE_DIST, "rb"))
    with tempfile.NamedTemporaryFile(suffix=".dist", delete=False) as f:      # the reference indexes its count tables with []
        pickle.dump({k: (defaultdict(int, v) if k != "word_casing_lookup" else v) for k, v in tables.items()}, f)
    try:
        tc = ns["TrueCaser"](f.name)
        cases, scores = T.truecase_differential_inputs(tables)
        g["truecase"] = {"cases": [tc.get_true_case(s, oov) for s, oov in cases], "scores": [tc.get_score(*x) for x in scores]}
    finally:
        os.unlink(f.name)

    out = os.path.join(ROOT, "tests", "golden", "api_reference.json")
    json.dump(g, open(out, "w"), separators=(",", ":"), sort_keys=True, default=lambda x: x.item() if isinstance(x, np.generic) else str(x))
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
