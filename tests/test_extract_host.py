"""Fields out of forms on the CPU (yomitoku_b200/extractor.py, extract.py):

  * the extractor against tests/golden/extract_ref.json: the reference's own rule-based extractor on the same pages
    and schemas (tests/golden/make_golden_extract.py), in both output forms;
  * the literal expectations of the reference's extractor tests for the normalisers, the schema and the
    normalisation of resolved fields, carried over as data;
  * schema validation errors;
  * the command line with the suite's stand-in TableSemanticParser (tsp_cases.standin_parser, the word assignment as
    the oracle's Python loop): file names, --pages, --batch, --simple, --no-normalize, --encoding and the refusals."""
import importlib
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
from pydantic import ValidationError

import yomitoku_b200
from tsp_cases import load_cases, oracle_assign, standin_parser
from yomitoku_b200 import TableSemanticParser, extract
from yomitoku_b200 import extractor as ex
from yomitoku_b200.schemas import TableSemanticParserSchema

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
SCHEMAS = os.path.join(GOLDEN, "extract_schemas")
with open(os.path.join(GOLDEN, "extract_ref.json"), encoding="utf-8") as _f:
    REF = json.load(_f)
CASES = REF["cases"]


# ------------------------------------------------------------------------------------------------ the golden
@pytest.mark.parametrize("case", CASES, ids=["%s-%s" % (c["page"], c["schema"]) for c in CASES])
def test_extract_equals_reference(case):
    page = TableSemanticParserSchema.model_validate(REF["pages"][case["page"]])
    schema = ex.ExtractionSchema.from_yaml(os.path.join(SCHEMAS, case["schema"]))
    assert extract(page, schema, normalize=False) == case["full"]
    assert extract(page, schema, normalize=False, simple=True) == case["simple"]


def test_golden_pages_are_the_reference_dumps_with_texts():
    for name, page in REF["pages"].items():
        if name == "text_page":
            continue
        with open(os.path.join(GOLDEN, "table_semantic_outputs", name), encoding="utf-8") as f:
            source = json.load(f)
        blank = json.loads(json.dumps(page))
        for table in blank["tables"]:
            for cell in table["cells"].values():
                cell["contents"] = ""
        assert blank == source, name


def test_golden_reaches_every_path():
    sources = [f["source"] for c in CASES for f in c["full"]["fields"].values()]
    assert {"cell_id", "bbox", "kv", "cell_query", "paragraph", "regex", "not_found", "grid"} <= set(sources)
    full = {(c["page"], c["schema"]): c["full"]["fields"] for c in CASES}
    app = full[("debug_table_raw_10.golden.json", "application.yaml")]
    assert app["emails"]["cell_ids"] == ["r1c1", "r2c0"] and app["emails"]["source"] == "kv"        # merged, by y
    assert full[("debug_table_raw_0.golden.json", "application.yaml")]["row_keys"]["value"].count(",") == 2  # by x
    txt = full[("text_page", "application.yaml")]
    assert txt["invoice_number"]["cell_ids"] == ["w2"]                                            # a word
    assert txt["tel_number"]["cell_ids"] == ["p2"] and txt["address_paragraph"]["cell_ids"] == ["p0"]
    # a group cell's text is not searched
    assert full[("debug_table_raw_6.golden.json", "application.yaml")]["invoice_number"]["source"] == "not_found"
    items = full[("debug_table_raw_10.golden.json", "items.yaml")]
    assert len(items["items"]["records"]) == 5                                  # the header row is skipped
    assert items["yen_columns"]["records"][0]["yen"]["cell_ids"] == ["r5c1", "r5c2"]


# ------------------------------------------------------------------------------------------------ normalisers
# (rule, input, expected) of the reference's tests/test_extractor.py
NORMALIZER_EXPECTATIONS = [
    ("strip_spaces", "東京都　渋谷区", "東京都渋谷区"), ("strip_spaces", "a b c", "abc"), ("strip_spaces", "hello", "hello"),
    ("numeric", "１，２３４円", "1234"), ("numeric", "¥3,000", "3000"), ("numeric", "-100.5", "-100.5"),
    ("phone_jp", "０９０１２３４５６７８", "090-1234-5678"), ("phone_jp", "０３１２３４５６７８", "031-234-5678"),
    ("postal_code_jp", "１２３４５６７", "123-4567"), ("postal_code_jp", "123-4567", "123-4567"),
    ("date_jp", "令和6年3月15日", "2024-03-15"), ("date_jp", "平成30年1月1日", "2018-01-01"),
    ("date_jp", "昭和60年12月25日", "1985-12-25"), ("date_jp", "R6/3/15", "2024-03-15"),
    ("date_jp", "H30.1.1", "2018-01-01"), ("date_jp", "S60-12-25", "1985-12-25"), ("date_jp", "R5年1月11日", "2023-01-11"),
    ("date_jp", "2024年3月15日", "2024-03-15"), ("date_jp", "2024/3/15", "2024-03-15"),
    ("date_jp", "2024-03-15", "2024-03-15"), ("date_jp", "不明な日付", "不明な日付"),
    ("date_jp", "明治45年7月30日", "1912-07-30"), ("date_jp", "大正15年12月25日", "1926-12-25"),
    ("date_jp", "T15/12/25", "1926-12-25"), ("date_jp", "M45.7.30", "1912-07-30"),
    ("date_jp", "令和６年３月１５日", "2024-03-15"),
    ("date_yyyymmdd", "令和6年3月15日", "20240315"), ("date_yyyymmdd", "R5/01/11", "20230111"),
    ("date_yyyymmdd", "2024/3/15", "20240315"),
    ("time_jp", "14:30", "14時30分"), ("time_jp", "9:05:30", "9時05分30秒"), ("time_jp", "14時30分", "14時30分"),
    ("time_jp", "１４：３０", "14時30分"),
    ("time_hms", "14時30分", "14:30:00"), ("time_hms", "9:5", "09:05:00"), ("time_hms", "14:30:59", "14:30:59"),
    ("time_hms", "１４時３０分", "14:30:00"),
    ("alphanumeric", "ＡＢＣ１２３", "ABC123"), ("alphanumeric", "abc 123!@#", "abc123"), ("alphanumeric", "商品A01", "A01"),
    ("hiragana", "カタカナ", "かたかな"), ("hiragana", "ひらがな", "ひらがな"), ("hiragana", "テスト123abc", "てすと"),
    ("hiragana", "カタカナとひらがな混在", "かたかなとひらがな"),
    ("katakana", "ひらがな", "ヒラガナ"), ("katakana", "カタカナ", "カタカナ"), ("katakana", "テスト123abc", "テスト"),
    ("katakana", "ひらがなとカタカナ混在", "ヒラガナトカタカナ"),
]
# (value, rule, expected) of apply_normalize
APPLY_EXPECTATIONS = [("hello", None, "hello"), ("hello", "unknown_rule", "hello"), ("１２３", "numeric", "123"),
                      (12345, "phone_jp", "12345"), (12345, None, "12345"), (100, "numeric", "100")]


@pytest.mark.parametrize("rule,text,want", NORMALIZER_EXPECTATIONS)
def test_normalizer(rule, text, want):
    assert ex.NORMALIZERS[rule](text) == want
    assert ex.apply_normalize(text, rule) == want


@pytest.mark.parametrize("value,rule,want", APPLY_EXPECTATIONS)
def test_apply_normalize(value, rule, want):
    assert ex.apply_normalize(value, rule) == want


def test_registered_rules():
    assert sorted(ex.NORMALIZERS) == sorted(["strip_spaces", "numeric", "phone_jp", "postal_code_jp", "date_jp",
                                             "date_yyyymmdd", "time_jp", "time_hms", "alphanumeric", "hiragana",
                                             "katakana"])


def test_character_conversions():
    full = "".join(chr(c) for c in range(0xFF01, 0xFF5F)) + "　"
    assert ex.full_to_half(full) == "".join(chr(c) for c in range(0x21, 0x7F)) + " "
    assert ex.full_to_half("￥ｶﾞ〜") == "￥ｶﾞ〜"                      # outside the two ranges: unchanged
    kata = "".join(chr(c) for c in range(0x30A1, 0x30F7))
    hira = "".join(chr(c) for c in range(0x3041, 0x3097))
    assert ex.kata_to_hira(kata) == hira and ex.hira_to_kata(hira) == kata
    assert ex.kata_to_hira("ーヷヽ") == "ーヷヽ" and ex.hira_to_kata("ゝゞ") == "ゝゞ"
    assert ex.NORMALIZERS["katakana"]("らーめん") == "ラーメン"
    assert ex.NORMALIZERS["hiragana"]("ラーメン") == "らめん"           # ー is not in the hiragana block


# ------------------------------------------------------------------------------------------------ schema
# (YAML, [(field index, attribute, expected)]) of the reference's tests/test_extractor.py
SCHEMA_EXPECTATIONS = [
    ("fields:\n  - name: phone\n    description: 電話番号\n    type: string\n    normalize: phone_jp\n"
     "  - name: amount\n    description: 合計金額\n    type: number\n    normalize: numeric\n",
     [(0, "name", "phone"), (0, "description", "電話番号"), (0, "type", "string"), (0, "normalize", "phone_jp"),
      (0, "structure", "scalar"), (1, "type", "number")]),
    ("fields:\n  - name: f1\n    cell_id: c12\n    type: string\n  - name: f2\n    bbox: [100, 200, 300, 400]\n"
     "    type: string\n  - name: f3\n    regex: 'T\\d{13}'\n    type: string\n",
     [(0, "cell_id", "c12"), (1, "bbox", [100, 200, 300, 400]), (2, "regex", r"T\d{13}")]),
    ("fields:\n  - name: phone\n    description: 電話番号\n    structure: kv\n    type: string\n",
     [(0, "structure", "kv"), (0, "merge_values", False), (0, "separator", "\n"), (0, "columns", None)]),
]
TABLE_SCHEMA = ("fields:\n  - name: items\n    structure: table\n    columns:\n      - name: product\n"
                "        description: 商品名\n        type: string\n      - name: price\n        description: 金額\n"
                "        type: number\n        normalize: numeric\n      - name: col1\n        cell_id: c5\n"
                "      - name: col2\n        bbox: [10, 20, 30, 40]\n")


@pytest.mark.parametrize("i", range(len(SCHEMA_EXPECTATIONS)))
def test_schema_from_yaml(tmp_path, i):
    text, checks = SCHEMA_EXPECTATIONS[i]
    p = tmp_path / "schema.yaml"
    p.write_text(text, encoding="utf-8")
    schema = ex.ExtractionSchema.from_yaml(str(p))
    for idx, attr, want in checks:
        assert getattr(schema.fields[idx], attr) == want


def test_table_schema_from_yaml(tmp_path):
    p = tmp_path / "schema.yaml"
    p.write_text(TABLE_SCHEMA, encoding="utf-8")
    f = ex.ExtractionSchema.from_yaml(str(p)).fields[0]
    assert f.structure == "table" and len(f.columns) == 4
    assert (f.columns[0].name, f.columns[1].normalize, f.columns[2].cell_id, f.columns[3].bbox) == \
        ("product", "numeric", "c5", [10, 20, 30, 40])
    assert f.columns[0].type == "string" and f.columns[2].description == "" and f.columns[2].type == "string"


@pytest.mark.parametrize("data,loc", [
    ({"fields": [{"name": "a", "structure": "list"}]}, ("fields", 0, "structure")),
    ({"fields": [{"description": "no name"}]}, ("fields", 0, "name")),
    ({"fields": [{"name": "a", "type": "money"}]}, ("fields", 0, "type")),
    ({"fields": [{"name": "a", "bbox": "top left"}]}, ("fields", 0, "bbox")),
    ({"fields": [{"name": "t", "structure": "table", "columns": [{"description": "x"}]}]},
     ("fields", 0, "columns", 0, "name")),
    ({"fields": [{"name": "t", "structure": "table", "columns": [{"name": "c", "type": "list"}]}]},
     ("fields", 0, "columns", 0, "type")),
    ({}, ("fields",)),
])
def test_schema_errors_name_the_field(data, loc):
    with pytest.raises(ValidationError) as e:
        ex.ExtractionSchema.model_validate(data)
    assert loc in [err["loc"] for err in e.value.errors()]
    assert loc[-1] in str(e.value)


def test_as_schema(tmp_path):
    p = tmp_path / "s.yaml"
    p.write_text("fields:\n  - name: a\n", encoding="utf-8")
    s = ex.as_schema(str(p))
    assert ex.as_schema(s) is s and ex.as_schema({"fields": [{"name": "a"}]}) == s
    with pytest.raises(ValidationError):
        ex.as_schema({"fields": [{"name": "a", "structure": "tree"}]})


# ------------------------------------------------------------------------------------------------ normalisation
def _schema(fields):
    return ex.ExtractionSchema.model_validate({"fields": fields})


@pytest.mark.parametrize("field,skip,want", [
    ({"name": "phone", "type": "string", "normalize": "phone_jp"}, False, "090-1234-5678"),
    ({"name": "phone", "type": "string", "structure": "kv", "normalize": "phone_jp"}, False, "090-1234-5678"),
    ({"name": "phone", "type": "string", "normalize": "phone_jp"}, True, "09012345678"),
])
def test_normalize_scalar_fields(field, skip, want):
    fields = [ex.ResolvedField(name="phone", value="09012345678", raw_text="09012345678")]
    if not skip:
        ex.normalize_fields(fields, _schema([field]))
    assert fields[0].value == want


def test_normalize_table_columns():
    schema = _schema([{"name": "items", "structure": "table",
                       "columns": [{"name": "price", "type": "number", "normalize": "numeric"}]}])
    fields = [ex.ResolvedField(name="items", value=[{"price": {"value": "１，２００円", "cell_ids": ["c1"]}}],
                               raw_text="")]
    assert ex.normalize_fields(fields, schema)[0].value[0]["price"]["value"] == "1200"


def test_extract_normalizes_the_golden_page():
    page = TableSemanticParserSchema.model_validate(REF["pages"]["debug_table_raw_10.golden.json"])
    out = extract(page, os.path.join(SCHEMAS, "application.yaml"), simple=True)
    raw = extract(page, os.path.join(SCHEMAS, "application.yaml"), normalize=False, simple=True)
    assert (out["applicant"], raw["applicant"]) == ("山田太郎", "山田 太郎")
    assert out["phone"] == "031-234-5678"                       # ten digits: 3-3-4, as the reference
    assert out["postal"] == "150-0002"
    assert out["cell_id_missing_then_key"] == "2024-03-15"
    assert out["visit_time"] == "14:30:00"
    items = extract(page, os.path.join(SCHEMAS, "items.yaml"))["fields"]["items"]["records"]
    assert [r["amount"]["value"] for r in items] == ["1200", "500", "", "100", "1800"]
    assert items[0]["amount"]["raw_text"] == "１，２００円"      # the cell's own text stays beside the value


def test_build_outputs():
    fields = [ex.ResolvedField("phone", "03-1234-5678", "0312345678",
                               [ex.ResolvedElement("c1", [10, 20, 30, 40], "0312345678")], "high", "kv"),
              ex.ResolvedField("items", [{"product": {"value": "apple", "cell_ids": ["c1"]},
                                          "price": {"value": "100", "cell_ids": ["c2"]}}], "",
                               [ex.ResolvedElement("c1", [0, 0, 50, 30], "apple"),
                                ex.ResolvedElement("c2", [50, 0, 100, 30], "100")], "high", "grid"),
              ex.ResolvedField("model_code", {"value": "100031582200", "cell_ids": ["c6"]}, "")]
    full = ex.build_output(fields[:2])
    assert full["metadata"] == {"schema_version": "1.0"}
    assert full["fields"]["phone"] == {"structure": "kv", "value": "03-1234-5678", "raw_text": "0312345678",
                                       "confidence": "high", "source": "kv", "cell_ids": ["c1"],
                                       "bboxes": [[10, 20, 30, 40]]}
    rec = full["fields"]["items"]["records"][0]
    assert rec["product"] == {"value": "apple", "cell_ids": ["c1"], "raw_text": "apple", "bboxes": [[0, 0, 50, 30]]}
    assert ex.build_simple_output(fields) == {"phone": "03-1234-5678", "items": [{"product": "apple", "price": "100"}],
                                              "model_code": "100031582200"}


def test_search_cells_by_query():
    page = TableSemanticParserSchema.model_validate(REF["pages"]["debug_table_raw_10.golden.json"])
    t0 = page.tables[0]
    assert [c.id for c in t0.search_cells_by_query("氏 名")] == ["r1c0"]
    assert [c.id for c in t0.search_cells_by_query("（円）")] == ["r4c2", "r4c3"]
    assert t0.search_cells_by_query("存在しない") == []
    page6 = TableSemanticParserSchema.model_validate(REF["pages"]["debug_table_raw_6.golden.json"])
    assert page6.tables[0].search_cells_by_query("T0000000000000") == []          # group cells are not searched


# ------------------------------------------------------------------------------------------------ command line
TSP_CASES = load_cases()
# the command line module; `yomitoku_b200.extract` is also the package's extract function, so `from yomitoku_b200
# import extract` gives the function
cli = importlib.import_module("yomitoku_b200.extract")
CLI_SCHEMA = """fields:
  - name: 番号
    regex: '[0-9]{2}'
  - name: first_header
    cell_id: r0c0
  - name: code
    regex: '[a-z][0-9]'
    normalize: alphanumeric
  - name: grid
    structure: table
    columns:
      - name: 見出し
        cell_id: r0c0
      - name: second
        cell_id: r0c1
        normalize: katakana
"""


class StandinParser:
    """TableSemanticParser.extract_pages over the suite's stand-in parser: page i's semantic result is the golden
    table-semantic case chosen by the page's height, parsed by the product's host code."""

    extract_pages = TableSemanticParser.extract_pages

    def __init__(self):
        self.parsers = [standin_parser(c, device="cpu") for c in TSP_CASES]
        self.calls = []

    def semantic(self, page):
        return self.parsers[page.shape[0] % len(self.parsers)](page)[0]

    def parse_pages(self, pages):
        self.calls.append(len(pages))
        return [self.semantic(p) for p in pages]


@pytest.fixture
def parser(monkeypatch):
    from yomitoku_b200 import table_semantic_parser as tsp
    monkeypatch.setattr(tsp, "assign_best_overlap", oracle_assign)
    return StandinParser()


def _page(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.fixture
def tree(tmp_path):
    """in/c.png (48x64), in/.hidden/a.png (40x50), in/sub/scan.tiff (3 frames of different sizes), schema.yaml."""
    from PIL import Image
    root = tmp_path / "in"
    (root / ".hidden").mkdir(parents=True)
    (root / "sub").mkdir()
    cv2.imwrite(str(root / "c.png"), _page(1, 48, 64))
    cv2.imwrite(str(root / ".hidden" / "a.png"), _page(2, 40, 50))
    frames = [Image.fromarray(_page(s, h, w)) for s, h, w in ((3, 41, 60), (4, 57, 36), (5, 33, 70))]
    frames[0].save(str(root / "sub" / "scan.tiff"), save_all=True, append_images=frames[1:])
    (tmp_path / "schema.yaml").write_text(CLI_SCHEMA, encoding="utf-8")
    return root


def _args(*argv):
    return cli.build_parser().parse_args([str(a) for a in argv])


def _run(*argv, parser):
    return cli.run(_args(*argv), parser)


def _pages_of(tree):
    from yomitoku_b200.data import load_image
    pages = {"a_p1": load_image(tree / ".hidden" / "a.png")[0], "c_p1": load_image(tree / "c.png")[0]}
    for i, p in enumerate(load_image(tree / "sub" / "scan.tiff")):
        pages["scan_p%d" % (i + 1)] = p
    return pages


@pytest.mark.parametrize("simple,normalize", [(False, True), (True, True), (False, False)])
def test_one_json_per_page(tree, tmp_path, parser, simple, normalize):
    out = tmp_path / "out"
    argv = [tree, "-s", tmp_path / "schema.yaml", "-o", out, "--batch", 2]
    argv += ["--simple"] if simple else []
    argv += ["--no-normalize"] if not normalize else []
    written = _run(*argv, parser=parser)
    names = ["a_p1", "c_p1", "scan_p1", "scan_p2", "scan_p3"]
    assert sorted(os.path.basename(w) for w in written) == ["%s_extract.json" % n for n in names]
    assert sorted(os.listdir(out)) == ["%s_extract.json" % n for n in names]
    assert parser.calls == [2, 2, 1]
    schema = str(tmp_path / "schema.yaml")
    for name, page in _pages_of(tree).items():
        want = ex.extract(parser.semantic(page), schema, normalize=normalize, simple=simple)
        text = (out / ("%s_extract.json" % name)).read_text(encoding="utf-8")
        assert text == json.dumps(want, ensure_ascii=False, indent=2)
        if simple:
            assert sorted(want) == sorted(["番号", "first_header", "code", "grid"])
        else:
            assert want["metadata"] == {"schema_version": "1.0"} and "番号" in want["fields"]
    # the pages reach more than one golden case, and the schema finds something on them
    outs = [json.loads((out / ("%s_extract.json" % n)).read_text(encoding="utf-8")) for n in names]
    assert len({json.dumps(o, sort_keys=True) for o in outs}) > 1
    if simple:
        assert any(o["番号"] for o in outs) and any(o["grid"] for o in outs)


def test_pages_and_encoding(tree, tmp_path, parser):
    out = tmp_path / "out"
    written = _run(tree / "sub" / "scan.tiff", "-s", tmp_path / "schema.yaml", "-o", out, "--pages", "1,3-5",
                   "--encoding", "shift-jis", "--simple", parser=parser)
    assert [os.path.basename(w) for w in written] == ["scan_p1_extract.json", "scan_p3_extract.json"]
    assert parser.calls == [2]
    pages = _pages_of(tree)
    raw = (out / "scan_p3_extract.json").read_bytes()
    assert "番号".encode("shift-jis") in raw and "番号".encode("utf-8") not in raw
    assert json.loads(raw.decode("shift-jis")) == ex.extract(parser.semantic(pages["scan_p3"]),
                                                             str(tmp_path / "schema.yaml"), simple=True)


def test_refusals_and_errors(tree, tmp_path, parser):
    schema = tmp_path / "schema.yaml"
    o = tmp_path / "o"
    with pytest.raises(ValueError, match="TrueType font"):
        _run(tree, "-s", schema, "-o", o, "-v", parser=parser)
    pdf = tmp_path / "doc.pdf"
    pdf.write_bytes(b"%PDF-1.4\n%%EOF\n")
    with pytest.raises(ValueError, match="PDF input is not supported"):
        _run(pdf, "-s", schema, "-o", o, parser=parser)
    with pytest.raises(FileNotFoundError, match="missing"):
        _run(tmp_path / "missing", "-s", schema, "-o", o, parser=parser)
    with pytest.raises(FileNotFoundError, match="Schema file not found"):
        _run(tree, "-s", tmp_path / "nope.yaml", "-o", o, parser=parser)
    bad = tmp_path / "bad.yaml"
    bad.write_text("fields:\n  - name: a\n    structure: tree\n", encoding="utf-8")
    with pytest.raises(ValidationError, match="structure"):
        _run(tree, "-s", bad, "-o", o, parser=parser)
    with pytest.raises(ValueError, match="Invalid encoding"):
        _run(tree, "-s", schema, "-o", o, "--encoding", "latin-1", parser=parser)
    with pytest.raises(ValueError, match="--batch"):
        _run(tree, "-s", schema, "-o", o, "--batch", "0", parser=parser)
    # refused before any model is built
    with pytest.raises(ValueError, match="TrueType font"):
        cli.main([str(tree), "-s", str(schema), "-v"])
    with pytest.raises(ValueError, match="PDF input is not supported"):
        cli.main([str(pdf), "-s", str(schema)])
    with pytest.raises(FileNotFoundError, match="Schema file not found"):
        cli.main([str(tree), "-s", str(tmp_path / "nope.yaml")])
    with pytest.raises(SystemExit):
        _args(tree)                                     # -s is required
    with pytest.raises(SystemExit):
        _args(tree, "-s", schema, "--dpi", "300")
    assert parser.calls == [] and not o.exists()


def test_unreadable_files_are_skipped(tree, tmp_path, parser):
    (tree / "broken.png").write_bytes(b"not an image")
    (tree / "notes.txt").write_text("hello")
    (tree / "doc.pdf").write_bytes(b"%PDF-1.4\n%%EOF\n")
    written = _run(tree, "-s", tmp_path / "schema.yaml", "-o", tmp_path / "out", parser=parser)
    assert sorted(os.path.basename(w) for w in written) == [
        "a_p1_extract.json", "c_p1_extract.json", "scan_p1_extract.json", "scan_p2_extract.json",
        "scan_p3_extract.json"]
    assert parser.calls == [5]


def test_defaults_and_configs():
    a = _args("x", "-s", "s.yaml")
    assert (a.outdir, a.device, a.batch, a.encoding, a.cell_detector_model, a.pages, a.simple, a.no_normalize,
            a.vis) == ("results", "cuda", 16, "utf-8", "rtdetrv2", None, False, False, False)
    assert cli.parser_configs(a) == {"table_cell_parser": {"model_name": "rtdetrv2"}}
    assert cli.parser_configs(_args("x", "-s", "s.yaml", "-l"))["text_recognizer"] == {
        "model_name": "parseq-tiny-dynw-v4", "dynamic_width": True, "batch_bucketing": True}


def test_module_entry_point():
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-m", "yomitoku_b200.extract", "--help"], cwd=root, capture_output=True,
                       text=True)
    assert r.returncode == 0 and "--schema" in r.stdout and "--batch" in r.stdout and "--simple" in r.stdout


def test_package_extract_stays_callable_after_the_command_line_module_is_imported():
    page = TableSemanticParserSchema.model_validate(REF["pages"]["text_page"])
    schema = {"fields": [{"name": "heading", "description": "請求書"}]}
    assert yomitoku_b200.extract is cli
    assert yomitoku_b200.extract(page, schema, simple=True) == extract(page, schema, simple=True) == {"heading": "請求書"}
