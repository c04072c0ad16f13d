"""The get-entries body rules of tests/bodies_oracle.py: one test per rule, agreement with Python's json where the two
agree, with find_entry_spans on the bodies get_entries_body writes, and the Go scanner's silent drop on '": "'."""
import json
import random

import pytest

import bodies_oracle as bo
from ct_mapreduce_b200 import frontend

OK, BAD_JSON, BAD_TYPE, TOO_MANY, REPEATED = (bo.BODY_OK, bo.BODY_BAD_JSON, bo.BODY_BAD_TYPE, bo.BODY_TOO_MANY,
                                              bo.BODY_REPEATED_ENTRIES)


def st(body, mx=10):
    return bo.parse_body(body, mx)[0]


def datas(body, mx=10):
    s, ents = bo.parse_body(body, mx)
    assert s == OK
    return [tuple(None if x is None else x.data for x in e) for e in ents]


@pytest.mark.parametrize("body", [b"", b" ", b"\xef\xbb\xbf{}", b"{", b"{}}", b"{} x", b"[1,]", b'{"a":1,}', b'{"a" 1}', b"{'a':1}",
                                  b"NaN", b"01", b"1.", b"-", b".5", b"1e", b"tru", b"nulll", b'"\x01"', b'"\\x"', b'"\\u12g4"',
                                  b'"abc', b"{}\x0b", b'{"entries":[]}\x00'])
def test_bad_json(body):
    assert st(body) == BAD_JSON


@pytest.mark.parametrize("body", [b"null", b"{}", b" \t\r\n{}\n", b'{"x":[1,-0.5e+3,true,false,null,{"y":{}}]}', b'{"a":"\xff"}',
                                  b'{"entries":null}', b'{"entries":[]}'])
def test_valid_bodies_without_entries(body):
    assert bo.parse_body(body, 0) == (OK, [])


@pytest.mark.parametrize("body", [b"[]", b"1", b'"s"', b"true", b'{"entries":{}}', b'{"entries":"x"}', b'{"entries":[1]}',
                                  b'{"entries":[[]]}', b'{"entries":[{"leaf_input":1}]}', b'{"entries":[{"extra_data":{}}]}',
                                  b'{"entries":[{"leaf_input":[]}]}'])
def test_bad_type(body):
    assert st(body) == BAD_TYPE


def test_whitespace_everywhere_and_key_order():
    body = b' {\n "entries" : [ { "extra_data" : "QQ==" , "leaf_input" : "AAAA" } ] } '
    assert datas(body) == [(b"AAAA", b"QQ==")]


def test_missing_repeated_and_null_keys():
    assert datas(b'{"entries":[{"leaf_input":"AAAA"}]}') == [(b"AAAA", None)]
    assert datas(b'{"entries":[{"leaf_input":"AAAA","leaf_input":"BBBB","extra_data":"CC==","extra_data":null}]}') == [(b"BBBB", None)]
    assert datas(b'{"entries":[null,{}]}') == [(None, None), (None, None)]


def test_case_folded_keys():
    assert datas(b'{"ENTRIES":[{"Leaf_Input":"AAAA","EXTRA_data":"BBBB"}]}') == [(b"AAAA", b"BBBB")]
    assert datas(b'{"entries":[{"leafinput":"AAAA","leaf-input":"BBBB"}]}') == [(None, None)]  # '_' is exact


def test_entries_long_s():
    assert datas('{"entrieſ":[{"leaf_input":"AAAA"}]}'.encode()) == [(b"AAAA", None)]
    assert datas(b'{"entrie\\u017f":[{"leaf_input":"AAAA"}]}') == [(b"AAAA", None)]
    assert bo.parse_body('{"entrieſ":[]}'.encode().replace(b"\xc5\xbf", b"\xc5"), 1) == (OK, [])  # no entries key


def test_escaped_keys_and_base64():
    body = b'{"ent\\u0072ies":[{"leaf\\u005finput":"AA\\/A\\nBB\\u0042B","extra_data":"A\\u00e9=="}]}'
    s, ents = bo.parse_body(body, 1)
    assert s == OK
    leaf, extra = ents[0]
    assert leaf.escaped and leaf.data == b"AA/ABBBB" and body[leaf.off:leaf.off + leaf.len] == b"AA\\/A\\nBB\\u0042B"
    assert extra.data == b"A!!=="  # each byte of the non-ASCII character: outside the alphabet


def test_deep_unknown_fields_holding_the_key_names():
    body = (b'{"x":{"entries":[{"leaf_input":"ZZZZ"}]},"entries":[{"y":{"leaf_input":"ZZZZ","extra_data":[]},'
            b'"leaf_input":"AAAA","z":[[[{"extra_data":"ZZZZ"}]]]}],"w":' + b"[" * 200 + b"]" * 200 + b"}")
    assert datas(body) == [(b"AAAA", None)]


def test_too_many_and_repeated():
    one = b'{"leaf_input":"AAAA","extra_data":"BBBB"}'
    assert st(b'{"entries":[' + b",".join([one] * 3) + b"]}", 2) == TOO_MANY
    assert st(b'{"entries":[' + b",".join([one] * 3) + b"]}", 3) == OK
    assert st(b'{"entries":[],"Entries":[]}') == REPEATED
    assert st(b'{"entries":[],"Entries":[1]}') == BAD_TYPE     # types are checked in the later array too
    assert st(b'{"entries":[],"Entries":[1}') == BAD_JSON


def test_agrees_with_python_json():
    rng = random.Random(11)
    for _ in range(400):
        ents = [{"leaf_input": "QUFB" * rng.randrange(3), "extra_data": "QkJC" * rng.randrange(3)} for _ in range(rng.randrange(4))]
        doc = {"entries": ents, "other": {"n": rng.random(), "l": [None, True, "leaf_input"]}}
        body = json.dumps(doc, indent=rng.choice([None, 1, 2]), separators=rng.choice([None, (",", ":")])).encode()
        assert datas(body) == [(e["leaf_input"].encode(), e["extra_data"].encode()) for e in ents]
    for body in (b'{"a":1e400}', b'[1, 2', b'{"a" : tru}', b'{"a":"\\ud800"}', b'{"a":"\t"}'):
        try:
            json.loads(body, strict=True)
            ok = True
        except ValueError:
            ok = False
        assert (st(body) != BAD_JSON) == ok, body


def test_agrees_with_find_entry_spans():
    rng = random.Random(5)
    pairs = [(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 60))), bytes(rng.randrange(256) for _ in range(rng.randrange(0, 60))))
             for _ in range(50)]
    body = frontend.get_entries_body(pairs)
    lo, ll, xo, xl = frontend.find_entry_spans(body)
    s, ents = bo.parse_body(body, 50)
    assert s == OK
    assert [(e[0].off, e[0].len, e[1].off, e[1].len) for e in ents] == list(zip(lo.tolist(), ll.tolist(), xo.tolist(), xl.tolist()))


def test_go_scanner_drops_a_spaced_body_silently_and_the_oracle_does_not():
    body = b'{"entries":[{"leaf_input": "AAAA","extra_data": "BBBB"}]}'
    assert bo.go_scanner_spans(body) == []          # equal counts (zero and zero): no error, no entry
    assert datas(body) == [(b"AAAA", b"BBBB")]


def test_twin_batch_places_unescaped_strings_after_the_bodies():
    bodies = [b'{"entries":[{"leaf_input":"A\\u0041AA","extra_data":"BBBB"}]}', b"{}", b"x"]
    text, lo, ll, xo, xl, sts, cnts = bo.twin_batch(bodies, [1, 1, 1])
    assert sts == [OK, OK, BAD_JSON] and cnts == [1, 0, 0]
    assert text[lo[0]:lo[0] + ll[0]] == b"AAAA" and text[xo[0]:xo[0] + xl[0]] == b"BBBB"
