"""Generates tests/golden/extract_ref.json: what the reference's rule-based extractor (`run_rule_extraction`,
src/yomitoku/extractor/rule_pipeline.py with its schema.py, resolver.py and pipeline.py) returns for every page below
and every schema in tests/golden/extract_schemas/, with no_normalize=True, in the full and the simple output form.
The reference's files are executed from /root/reference by path (build container only), on top of the table semantic
parser modules make_golden_tsp.py loads the same way; the modules the extractor imports but this path never executes
(the LLM client, the prompt builder, the visualiser) are stubs.

The reference's normaliser imports `jaconv`, which is not installed: a stand-in module takes the import, and its
functions raise, so that nothing in the golden comes from it (normalisation is off).

Pages: three of the reference's own TableSemanticParser dumps (tests/golden/table_semantic_outputs/, copied from the
reference's tests/data/table_semantic_outputs/; their cells have no text) with texts written into their cells, plus
one page of paragraphs and words.  The reference orders key-value items by set iteration in places, so the generator
runs it under three hash seeds and requires the outputs to agree.
Usage: python tests/golden/make_golden_extract.py
"""
import copy
import glob
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
SCHEMAS = os.path.join(HERE, "extract_schemas")
SOURCES = os.path.join(HERE, "table_semantic_outputs")

# ------------------------------------------------------------------------------------------------ pages
# cell texts per source dump: [table index][cell id] (cells not listed keep "")
TEXTS = {
    "debug_table_raw_10.golden.json": [
        {"r0c0": "申込者情報", "r1c0": "氏　名", "r1c1": "山田 太郎", "r2c0": "電話番号",
         "r2c1": "０３－１２３４－５６７８", "r3c0": "郵便番号", "r3c1": "〒１５０－０００２",
         "r4c0": "明細", "r4c1": "品名", "r4c2": "単価（円）", "r4c3": "金額（円）",
         "r5c0": "りんご", "r5c1": "１２０", "r5c2": "１，２００円",
         "r6c0": "みかん", "r6c1": "50", "r6c2": "500円",
         "r8c0": "登録番号T1234567890123", "r8c1": "1", "r8c2": "100",
         "r9c0": "小計", "r9c2": "1,800円"},
        {"r0c0": "連絡先", "r1c0": "メール", "r1c1": "taro@example.com", "r2c0": "hanako@example.com",
         "r3c0": "住所", "r3c1": "東京都渋谷区1-2-3", "r4c0": "サンプルビル5F", "r5c0": "申込日",
         "r5c1": "令和6年3月15日", "r6c0": "受付時刻", "r6c1": "14時30分"},
    ],
    "debug_table_raw_0.golden.json": [
        {"r0c0": "区分", "r0c1": "品名", "r0c2": "単価", "r0c3": "数量", "r0c4": "金額", "r0c5": "備考",
         "r1c0": "A", "r1c1": "ボールペン", "r1c2": "１２０", "r1c3": "3", "r1c4": "360", "r1c5": "至急"},
        {"r0c0": "区分", "r0c1": "区分", "r1c0": "一", "r1c1": "二", "r2c0": "三", "r2c1": "四",
         "r3c0": "五", "r3c1": "六", "r4c0": "七", "r4c1": "八", "r5c0": "左の値", "r5c1": "右の値"},
    ],
    "debug_table_raw_6.golden.json": [
        {"r0c0": "会社名", "r0c1": "株式会社サンプル", "r1c0": "担当者", "r1c1": "佐藤 花子", "r2c0": "電話",
         "r2c1": "090-1234-5678", "r3c0": "郵便番号", "r3c1": "1234567", "grp0": "T0000000000000"},
    ],
}


def _quad(x1, y1, x2, y2):
    return [[x1, y1], [x2, y1], [x2, y2], [x1, y2]]


def _word(text, box):
    return {"points": _quad(*box), "content": text, "direction": "horizontal", "rec_score": 0.9, "det_score": 0.8}


TEXT_PAGE = {
    "tables": [],
    "paragraphs": [
        {"id": "p0", "box": [100, 50, 600, 110], "contents": "請求書", "score": 0.9, "role": "section_headings"},
        {"id": None, "box": [100, 150, 900, 200], "contents": "住所： 大阪府大阪市北区1-1", "score": 0.9,
         "role": None},
        {"id": "p2", "box": [100, 220, 900, 270], "contents": "TEL 06-1234-5678 受付 9:05", "score": 0.9,
         "role": None},
    ],
    "words": [_word("請求書", (100, 50, 600, 110)), _word("合計", (100, 300, 180, 340)),
              _word("T9876543210123", (200, 300, 500, 340)), _word("", (520, 300, 540, 340))],
}


def pages():
    """name -> TableSemanticParserSchema dump."""
    out = {}
    for name, texts in TEXTS.items():
        with open(os.path.join(SOURCES, name), encoding="utf-8") as f:
            page = json.load(f)
        for table, table_texts in zip(page["tables"], texts):
            for cid, text in table_texts.items():
                table["cells"][cid]["contents"] = text
        out[name] = page
    out["text_page"] = copy.deepcopy(TEXT_PAGE)
    return out


# ------------------------------------------------------------------------------------------------ the reference
def load_reference_extractor():
    from make_golden_tsp import _stub, load_reference_tsp
    from oracle import refcheck as rc
    load_reference_tsp()

    def not_here(*a, **k):
        raise AssertionError("the jaconv stand-in was called: the golden must not depend on it")
    _stub("jaconv", z2h=not_here, h2z=not_here, kata2hira=not_here, hira2kata=not_here)
    rc._pkg("ytk_ref.extractor")
    _stub("ytk_ref.extractor.llm_client", call_llm=None)
    _stub("ytk_ref.extractor.prompt", build_messages=None)
    _stub("ytk_ref.extractor.visualizer", extraction_visualizer=None)
    for mod in ("normalizer", "schema", "resolver", "pipeline"):
        rc._load("ytk_ref.extractor." + mod, "extractor/%s.py" % mod, "ytk_ref.extractor")
    return rc._load("ytk_ref.extractor.rule_pipeline", "extractor/rule_pipeline.py", "ytk_ref.extractor")


def child():
    rp = load_reference_extractor()
    ts = sys.modules["ytk_ref.schemas.table_semantic_parser"]
    schema_cls = sys.modules["ytk_ref.extractor.schema"].ExtractionSchema
    cases = []
    with tempfile.TemporaryDirectory() as tmp:
        for page_name, page in pages().items():
            for path in sorted(glob.glob(os.path.join(SCHEMAS, "*.yaml"))):
                schema = schema_cls.from_yaml(path)
                case = {"page": page_name, "schema": os.path.basename(path)}
                for form, simple in (("full", False), ("simple", True)):
                    info = ts.TableSemanticParserSchema.model_validate(page)
                    out = rp.run_rule_extraction(info, None, schema, no_normalize=True, simple=simple, outdir=tmp)
                    case[form] = json.loads(json.dumps(out, ensure_ascii=False))
                cases.append(case)
    json.dump(cases, sys.stdout, ensure_ascii=False)


def main():
    runs = []
    for hs in ("0", "1", "2"):
        env = dict(os.environ, PYTHONHASHSEED=hs, YTK_EXTRACT_CHILD="1")
        r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True)
        if r.returncode:
            raise SystemExit(r.stderr)
        runs.append(json.loads(r.stdout))
    assert runs[0] == runs[1] == runs[2], "the extraction depends on the string hash"
    with open(os.path.join(HERE, "extract_ref.json"), "w", encoding="utf-8") as f:
        json.dump({"pages": pages(), "cases": runs[0]}, f, ensure_ascii=False, indent=1)
    sources = {}
    for c in runs[0]:
        for form in ("full",):
            for fld in c[form]["fields"].values():
                sources[fld["source"]] = sources.get(fld["source"], 0) + 1
    print("wrote extract_ref.json: %d cases; field sources %s" % (len(runs[0]), json.dumps(sources, sort_keys=True)))


if __name__ == "__main__":
    child() if os.environ.get("YTK_EXTRACT_CHILD") == "1" else main()
