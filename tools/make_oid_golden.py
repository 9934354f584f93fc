#!/usr/bin/env python
"""Writes tests/golden/oid_classes.json from the reference's own dispatch: every `Type::NAME` in the match arms of
parse_cell_from_postgres_text (crates/etl/src/conversions/text.rs:28-173 of supabase/etl) is mapped to the ETL_K_*
class of its arm and to its oid (PostgreSQL's pg_type catalogue, the constants `postgres-types` generates its
`Type::NAME` items from).  Needs a checkout of the reference; the JSON is committed, so the tests do not.
Usage: python tools/make_oid_golden.py <supabase/etl checkout>"""
import json
import os
import re
import sys

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
SRC = os.path.join(sys.argv[1] if len(sys.argv) > 1 else ".", "crates/etl/src/conversions/text.rs")
# pg_type.dat: typname → oid for the names the reference dispatches on
PG = dict(BOOL=16, BYTEA=17, CHAR=18, NAME=19, INT8=20, INT2=21, INT4=23, TEXT=25, OID=26, JSON=114, FLOAT4=700, FLOAT8=701, MONEY=790,
          BPCHAR=1042, VARCHAR=1043, DATE=1082, TIME=1083, TIMESTAMP=1114, TIMESTAMPTZ=1184, NUMERIC=1700, UUID=2950, JSONB=3802,
          BOOL_ARRAY=1000, BYTEA_ARRAY=1001, CHAR_ARRAY=1002, NAME_ARRAY=1003, INT2_ARRAY=1005, INT4_ARRAY=1007, TEXT_ARRAY=1009,
          BPCHAR_ARRAY=1014, VARCHAR_ARRAY=1015, INT8_ARRAY=1016, FLOAT4_ARRAY=1021, FLOAT8_ARRAY=1022, OID_ARRAY=1028, JSON_ARRAY=199,
          MONEY_ARRAY=791, DATE_ARRAY=1182, TIME_ARRAY=1183, TIMESTAMP_ARRAY=1115, TIMESTAMPTZ_ARRAY=1185, NUMERIC_ARRAY=1231,
          UUID_ARRAY=2951, JSONB_ARRAY=3807)
K = dict(Bool=1, String=2, I16=3, I32=4, U32=5, I64=6, F32=7, F64=8, Numeric=9, Date=10, Time=11, Timestamp=12, TimestampTz=13,
         Uuid=14, Json=15, Bytes=16)
ARRAY = 0x20


def main():
    text = open(SRC).read()
    body = text[text.index("pub(crate) fn parse_cell_from_postgres_text"):text.index("fn parse_cell_from_postgres_text_array") if "fn parse_cell_from_postgres_text_array" in text else len(text)]
    body = body[body.index("match *typ"):] if "match *typ" in body else body[body.index("match"):]
    # split into arms at top-level "Type::X (| Type::Y)* =>"
    arms = re.findall(r"((?:Type::[A-Z0-9_]+\s*\|?\s*)+)=>(.*?)(?=\n\s*(?:Type::[A-Z0-9_]+|_ if|_ =>))", body, flags=re.S)
    classes = {}
    for names, rhs in arms:
        cell = re.search(r"Cell::([A-Za-z0-9]+)", rhs)
        arr = re.search(r"ArrayCell::([A-Za-z0-9]+)", rhs)
        for nm in re.findall(r"Type::([A-Z0-9_]+)", names):
            if arr:
                classes[PG[nm]] = ARRAY | K[arr.group(1)]
            else:
                classes[PG[nm]] = K[cell.group(1)]
    assert len(classes) == len(PG), (len(classes), len(PG))
    out = {"source": "crates/etl/src/conversions/text.rs:28-173 @ reference checkout", "classes": {str(k): v for k, v in sorted(classes.items())},
           # `_ if is_array_type(typ)` (text.rs:166-170): built-in array types without a typed arm, e.g. _interval, _inet, _xml, _int4range
           "other_builtin_arrays": [1187, 1041, 143, 3905, 651, 1270, 1561, 3221, 2949, 1006, 1013],
           # `_ =>` (text.rs:171) and unknown oids (utils.rs:11-13): interval, inet, xml, int4range, int2vector, oidvector, a user type
           "plain_text_examples": [1186, 869, 142, 3904, 22, 30, 16385, 0]}
    path = os.path.join(ROOT, "tests", "golden", "oid_classes.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path, len(classes), "typed oids")


if __name__ == "__main__":
    main()
