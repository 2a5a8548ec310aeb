"""Golden fixture for train.py's flags, defaults and store names, produced by running the REFERENCE's own parser and
store-name rule.

Run in the build container only (needs /root/reference, read-only):

    python tests/golden/make_golden_train_flags.py

Neither `agedb-dir/train.py` nor `imdb-wiki-dir/train.py` can be imported (the argv parse, tensorboard_logger and the
folder creation run at import time), so their module-level `parser = ...` / `parser.add_argument(...)` /
`parser.set_defaults(...)` statements and the store-name block (lines 78-93) are lifted out with `ast`, as
make_golden_metrics.py does, and executed unmodified.  Only data is written to train_flags.json: every option's
default, type, choices and nargs per script, and the parsed values and store name for a list of argv.
"""
import argparse
import ast
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPTS = {"agedb": "/root/reference/agedb-dir/train.py", "imdb_wiki": "/root/reference/imdb-wiki-dir/train.py"}

# store-name cases: each runs through the script of its --dataset (AgeDB-DIR's when none is given)
ARGV = [
    [],
    ["--lds"],
    ["--lds", "--lds_kernel", "triang"],
    ["--lds", "--lds_kernel", "laplace", "--lds_ks", "7", "--lds_sigma", "2"],
    ["--fds"],
    ["--fds", "--fds_kernel", "triang", "--fds_ks", "3", "--start_update", "1", "--start_smooth", "2"],
    ["--fds", "--lds", "--reweight", "sqrt_inv", "--fds_mmt", "0.5"],
    ["--reweight", "inverse"],
    ["--reweight", "sqrt_inv", "--retrain_fc", "--store_name", "run1"],
    ["--optimizer", "sgd", "--loss", "focal_l1", "--lr", "0.01", "--batch_size", "64", "--model", "resnet18"],
    ["--dataset", "agedb", "--fds", "--lds", "--reweight", "sqrt_inv"],
    ["--dataset", "imdb_wiki"],
    ["--dataset", "imdb_wiki", "--fds", "--lds", "--reweight", "sqrt_inv"],
    ["--dataset", "imdb_wiki", "--fds", "--lds", "--lds_ks", "9", "--fds_ks", "7", "--bucket_start", "3"],
    ["--dataset", "imdb_wiki", "--lds", "--lds_kernel", "laplace", "--loss", "mse", "--store_name", "x"],
]


def lift(path):
    """(parser, store-name statements) of one reference script."""
    tree = ast.parse(open(path).read())
    parser_stmts, name_stmts = [], []
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "parser" for t in node.targets):
            parser_stmts.append(node)
        elif (isinstance(node, ast.Expr) and isinstance(node.value, ast.Call)
              and isinstance(node.value.func, ast.Attribute) and isinstance(node.value.func.value, ast.Name)
              and node.value.func.value.id == "parser" and node.value.func.attr in ("add_argument", "set_defaults")):
            parser_stmts.append(node)
        elif isinstance(node, ast.If) and "args.store_name" in ast.unparse(node):
            name_stmts.append(node)
        elif isinstance(node, ast.Assign) and ast.unparse(node.targets[0]) == "args.store_name":
            name_stmts.append(node)
    ns = {"argparse": argparse}
    exec(compile(ast.Module(body=parser_stmts, type_ignores=[]), path, "exec"), ns)
    return ns["parser"], compile(ast.Module(body=name_stmts, type_ignores=[]), path, "exec")


def main():
    out = {"options": {}, "cases": []}
    lifted = {k: lift(p) for k, p in SCRIPTS.items()}
    for key, (parser, _) in lifted.items():
        opts = {}
        for a in parser._actions:
            if a.dest == "help":
                continue
            opts[a.dest] = {"flags": list(a.option_strings), "default": a.default,
                            "type": None if a.type is None else a.type.__name__,
                            "choices": None if a.choices is None else list(a.choices), "nargs": a.nargs,
                            "const": a.const}
        out["options"][key] = opts
    for argv in ARGV:
        key = "imdb_wiki" if "imdb_wiki" in argv else "agedb"
        parser, name_code = lifted[key]
        args, _ = parser.parse_known_args(argv)
        values = dict(vars(args))
        ns = {"args": args}
        exec(name_code, ns)
        out["cases"].append({"argv": argv, "script": key, "values": values, "store_name": args.store_name})
    with open(os.path.join(HERE, "train_flags.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    for c in out["cases"]:
        print(c["script"], c["argv"], c["store_name"])


if __name__ == "__main__":
    main()
