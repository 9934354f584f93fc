"""Type oid → decode class: the product's catalogue table (etl_b200/csrc/oid_classes.h, through the C ABI) and the
oracle's switch (oracle/oracle_cells.c) are two independent statements of text.rs:28-173 + utils.rs:7-16; both are
checked against tests/golden/oid_classes.json, extracted from the reference's own match arms by
tools/make_oid_golden.py (which needs a checkout of the reference, so its output is committed)."""
import json
import os

ROOT = os.path.normpath(os.path.join(os.path.dirname(__file__), ".."))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "oid_classes.json")))


def test_product_table_matches_reference_arms():
    from etl_b200 import abi
    lib = abi.load()
    for oid, cls in GOLD["classes"].items():
        assert lib.etl_dec_kind_for_type_oid(int(oid)) == cls, oid
    for oid in GOLD["other_builtin_arrays"]:
        assert lib.etl_dec_kind_for_type_oid(oid) == (0x20 | 2), oid     # ArrayCell::String (text.rs:166-170)
    for oid in GOLD["plain_text_examples"]:
        assert lib.etl_dec_kind_for_type_oid(oid) == 2, oid               # Cell::String (text.rs:171)


def test_oracle_switch_matches_reference_arms(oracle_mod):
    for oid, cls in GOLD["classes"].items():
        assert oracle_mod.kind_for_oid(int(oid)) == cls, oid
    for oid in GOLD["other_builtin_arrays"]:
        assert oracle_mod.kind_for_oid(oid) == (0x20 | 2), oid
    for oid in GOLD["plain_text_examples"]:
        assert oracle_mod.kind_for_oid(oid) == 2, oid


def test_product_and_oracle_agree_on_every_small_oid(oracle_mod):
    from etl_b200 import abi
    lib = abi.load()
    for oid in list(range(0, 8192)) + [16384, 70000, 2**32 - 1]:
        assert lib.etl_dec_kind_for_type_oid(oid) == oracle_mod.kind_for_oid(oid), oid
