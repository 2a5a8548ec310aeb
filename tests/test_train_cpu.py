"""train.py's flags, defaults and store names against the reference's own parsers (tests/golden/train_flags.json, made
by tests/golden/make_golden_train_flags.py from agedb-dir/train.py and imdb-wiki-dir/train.py).  With `--dataset
imdb_wiki` the driver must parse as imdb-wiki-dir/train.py does (LDS / FDS windows of 5 taps, FDS buckets from age
0), otherwise as agedb-dir/train.py; explicit flags still win.  No GPU needed."""
import json
import os

import pytest

from util import GOLDEN

FLAGS = json.load(open(os.path.join(GOLDEN, "train_flags.json")))
# options of train.py that the reference scripts do not have
OWN = {"synthetic", "device_transform", "device_decode"}


def train():
    import train as T
    return T


def parse(argv):
    return train().build_parser().parse_args(list(argv))


def dataset_argv(script):
    return [] if script == "agedb" else ["--dataset", script]


@pytest.mark.parametrize("script", ["agedb", "imdb_wiki"])
def test_options_match_the_reference_script(script):
    """Same option set; each option's type, choices, nargs and (for this --dataset) default, with the default's own
    Python type (`--lds_sigma` defaults to the int 1, so store names read `_1`)."""
    ref = FLAGS["options"][script]
    p = train().build_parser()
    mine = {a.dest: a for a in p._actions if a.dest != "help"}
    assert set(mine) - OWN == set(ref)
    args = vars(p.parse_args(dataset_argv(script)))
    for dest, want in ref.items():
        a = mine[dest]
        assert list(a.option_strings) == want["flags"], dest
        assert (None if a.type is None else a.type.__name__) == want["type"], dest
        assert (None if a.choices is None else list(a.choices)) == want["choices"], dest
        assert a.nargs == want["nargs"] and a.const == want["const"], dest
        if dest == "dataset":                       # one driver: its --dataset default stays AgeDB-DIR's
            assert args[dest] == script
            continue
        assert args[dest] == want["default"] and type(args[dest]) is type(want["default"]), dest


@pytest.mark.parametrize("case", FLAGS["cases"], ids=lambda c: " ".join(c["argv"]) or "defaults")
def test_parsed_values_and_store_name(case):
    args = parse(case["argv"])
    got = vars(args)
    for dest, want in case["values"].items():
        if dest == "augment":                       # parser.set_defaults(augment=True): read nowhere in the reference
            continue
        assert got[dest] == want and type(got[dest]) is type(want), dest
    assert train().store_name(args) == case["store_name"]


def test_store_name_keeps_literal_default_types():
    T = train()
    assert T.store_name(parse(["--lds"])) == "agedb_resnet50_lds_gau_9_1_adam_l1_0.001_256"
    assert T.store_name(parse(["--lds", "--lds_sigma", "1"])) == "agedb_resnet50_lds_gau_9_1.0_adam_l1_0.001_256"
    assert T.store_name(parse(["--dataset", "imdb_wiki", "--fds"])) == \
        "imdb_wiki_resnet50_fds_gau_5_1_0_1_0.9_adam_l1_0.001_256"


@pytest.mark.parametrize("argv,want", [
    ([], (9, 9, 3)),
    (["--dataset", "agedb"], (9, 9, 3)),
    (["--dataset", "imdb_wiki"], (5, 5, 0)),
    (["--dataset=imdb_wiki"], (5, 5, 0)),
    (["--dataset", "imdb_wiki", "--lds_ks", "9"], (9, 5, 0)),
    (["--dataset", "imdb_wiki", "--fds_ks", "3", "--bucket_start", "3"], (5, 3, 3)),
    (["--dataset", "agedb", "--bucket_start", "0", "--lds_ks", "5"], (5, 9, 0)),
])
def test_dataset_defaults_and_explicit_flags(argv, want):
    a = parse(argv)
    assert (a.lds_ks, a.fds_ks, a.bucket_start) == want


def test_defaults_do_not_leak_between_parses():
    p = train().build_parser()
    assert p.parse_args(["--dataset", "imdb_wiki"]).bucket_start == 0
    assert p.parse_args([]).bucket_start == 3


@pytest.mark.parametrize("argv", [
    ["--lds_kernel", "box"], ["--fds_kernel", "cosine"], ["--reweight", "sqrt"], ["--bucket_start", "1"],
    ["--dataset", "utk"], ["--optimizer", "rmsprop"], ["--loss", "bce"], ["--lds_ks", "5.0"],
])
def test_bad_values_are_refused(argv):
    with pytest.raises(SystemExit):
        parse(argv)
