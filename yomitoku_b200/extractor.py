"""Fields out of forms: yomitoku's rule-based extractor (`yomitoku_extract`; reference src/yomitoku/extractor/
{schema,normalizer,rule_pipeline,pipeline}.py) over the results of TableSemanticParser.

    schema = ExtractionSchema.from_yaml("invoice.yaml")
    out = extract(parser(page)[0], schema)                 # {"fields": {...}, "metadata": {"schema_version": "1.0"}}
    outs = parser.extract_pages(pages, schema, simple=True)   # one {name: value} per page, batched parse_pages

A schema lists fields.  A scalar (or "kv") field is looked up, first hit wins, by
  1. `cell_id`: that cell of the first table that has it;
  2. `bbox`: the first non-group cell more than half inside the box;
  3. `description` as a key: the value cell of the first key-value item whose key text contains it (spaces ignored);
     with `merge_values` and several hits, all value cells joined by `separator`, ordered top to bottom if their top
     edges spread at least as much as their left edges, else left to right;
  4. `description` as text: the first cell that contains it, then the first paragraph that contains it (spaces
     ignored);
  5. `regex`: the first match in a cell (group cells skipped), then in a paragraph, then in a word;
and is otherwise "not_found".  A table field maps each grid column to the first schema column whose `cell_id` is one
of the column's header cells, whose `bbox` covers more than half of one of them, or whose description (its name if it
has none) is contained in the header text; every grid row that is not made of header cells alone becomes a record.
Values are then normalised by the rules named in the schema (`normalize: postal_code_jp`, ...; NORMALIZERS).

The extraction is dictionary lookups and string tests over a few hundred cell texts per page: host code.  The models
and the word-to-cell assignment that produce those texts are the CUDA part (TableSemanticParser).
"""
import re
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Literal, Optional

import yaml
from pydantic import BaseModel, Field

from .document_analyzer import overlap_ratio, quad_to_xyxy

__all__ = ["ColumnSchema", "FieldSchema", "ExtractionSchema", "NORMALIZERS", "apply_normalize", "ResolvedElement",
           "ResolvedField", "resolve_fields", "normalize_fields", "build_output", "build_simple_output", "extract",
           "as_schema"]

SCHEMA_VERSION = "1.0"
ValueType = Literal["string", "number", "date", "alphanumeric", "hiragana", "katakana"]


# ------------------------------------------------------------------------------------------------ schema
class ColumnSchema(BaseModel):
    name: str = Field(..., description="Column name (the key of the column in each record)")
    description: str = Field("", description="Text looked for in the column's header")
    cell_id: Optional[str] = Field(None, description="Id of a header cell of the column")
    bbox: Optional[List[int]] = Field(None, description="[x1, y1, x2, y2] covering a header cell of the column")
    type: ValueType = Field("string", description="Value type")
    normalize: Optional[str] = Field(None, description="Normalisation rule name")


class FieldSchema(BaseModel):
    name: str = Field(..., description="Field name (the key of the field in the output)")
    description: str = Field("", description="Key text, or text the value's cell or paragraph contains")
    cell_id: Optional[str] = Field(None, description="Id of the value's cell")
    bbox: Optional[List[int]] = Field(None, description="[x1, y1, x2, y2] covering the value's cell")
    regex: Optional[str] = Field(None, description="Pattern the value matches")
    type: ValueType = Field("string", description="Value type (scalar fields)")
    structure: Literal["scalar", "kv", "table"] = Field("scalar", description="scalar (or kv) or table")
    normalize: Optional[str] = Field(None, description="Normalisation rule name (scalar fields)")
    merge_values: bool = Field(False, description="Join the values of every item whose key matches")
    separator: str = Field("\n", description="What joins merged values")
    columns: Optional[List[ColumnSchema]] = Field(None, description="Columns of a table field")


class ExtractionSchema(BaseModel):
    fields: List[FieldSchema] = Field(..., description="Fields to extract")

    @classmethod
    def from_yaml(cls, path):
        with open(path, "r", encoding="utf-8") as f:
            return cls.model_validate(yaml.safe_load(f))


def as_schema(schema):
    """An ExtractionSchema from an ExtractionSchema, a dict in its form or the path of a YAML file."""
    if isinstance(schema, ExtractionSchema):
        return schema
    if isinstance(schema, dict):
        return ExtractionSchema.model_validate(schema)
    return ExtractionSchema.from_yaml(schema)


# ------------------------------------------------------------------------------------------------ normalisers
_FULL_TO_HALF = {c: c - 0xFEE0 for c in range(0xFF01, 0xFF5F)}
_FULL_TO_HALF[0x3000] = 0x20
_KATA_TO_HIRA = {c: c - 0x60 for c in range(0x30A1, 0x30F7)}
_HIRA_TO_KATA = {c: c + 0x60 for c in range(0x3041, 0x3097)}


def full_to_half(text):
    """Full-width ASCII and digits (U+FF01-U+FF5E) to U+0021-U+007E, the ideographic space U+3000 to a space.
    Everything else is left as it is: half-width katakana, the full-width yen and cent signs (U+FFE5, U+FFE0), curly
    quotes and the wave dash among them."""
    return text.translate(_FULL_TO_HALF)


def kata_to_hira(text):
    """Katakana U+30A1-U+30F6 (ァ to ヶ) to the hiragana 0x60 below them; the long-vowel mark ー, ヷ-ヺ, the
    iteration marks and half-width katakana are left as they are."""
    return text.translate(_KATA_TO_HIRA)


def hira_to_kata(text):
    """Hiragana U+3041-U+3096 (ぁ to ゖ) to the katakana 0x60 above them; the iteration marks ゝゞ are left."""
    return text.translate(_HIRA_TO_KATA)


NORMALIZERS: Dict[str, Callable[[str], str]] = {}


def _rule(name):
    def register(fn):
        NORMALIZERS[name] = fn
        return fn
    return register


def apply_normalize(value, rule):
    """`value` as a string normalised by the rule named `rule`; None or an unknown rule gives str(value)."""
    text = value if isinstance(value, str) else str(value)
    fn = NORMALIZERS.get(rule) if rule is not None else None
    return fn(text) if fn is not None else text


@_rule("strip_spaces")
def strip_spaces(text):
    return re.sub(r"[\s\u3000]+", "", text)


@_rule("numeric")
def numeric(text):
    """Digits, ".", "-" and "+" only, after full-width to half-width ("１，２３４円" -> "1234")."""
    return re.sub(r"[^\d.\-+]", "", full_to_half(text).replace(",", "").replace("、", ""))


def _digits(text):
    return re.sub(r"[^\d]", "", full_to_half(text))


@_rule("phone_jp")
def phone_jp(text):
    """11 digits as 3-4-4, 10 digits as 3-3-4, any other count as the bare digits."""
    d = _digits(text)
    if len(d) == 11:
        return "%s-%s-%s" % (d[:3], d[3:7], d[7:])
    if len(d) == 10:
        return "%s-%s-%s" % (d[:3], d[3:6], d[6:])
    return d


@_rule("postal_code_jp")
def postal_code_jp(text):
    d = _digits(text)
    return "%s-%s" % (d[:3], d[3:]) if len(d) == 7 else d


# year 1 of each era is the offset + 1
_ERAS = (("令和", 2018), ("平成", 1988), ("昭和", 1925), ("大正", 1911), ("明治", 1867))
_ERA_LETTERS = {"R": 2018, "H": 1988, "S": 1925, "T": 1911, "M": 1867}
_YMD_KANJI = r"\s*(\d+)\s*年\s*(\d+)\s*月\s*(\d+)\s*日"


def _parse_date(text):
    """(year, month, day) of the first date form found, in this order: era name + 年月日 (令和6年3月15日), era letter +
    separated numbers (R6/3/15, H30.1.1, S60-12-25), era letter + 年月日 (R5年1月11日), 2024年3月15日, 2024/3/15 or
    2024-3-15; None if there is none.  Full-width digits count.  Day and month are not range-checked."""
    text = full_to_half(text)
    for era, offset in _ERAS:
        m = re.search(era + _YMD_KANJI, text)
        if m:
            return offset + int(m.group(1)), int(m.group(2)), int(m.group(3))
    for pattern in (r"([RHSTM])\s*(\d{1,2})\s*[/\-\.]\s*(\d{1,2})\s*[/\-\.]\s*(\d{1,2})",
                    r"([RHSTM])\s*(\d{1,2})\s*年\s*(\d{1,2})\s*月\s*(\d{1,2})\s*日"):
        m = re.search(pattern, text)
        if m:
            return _ERA_LETTERS[m.group(1)] + int(m.group(2)), int(m.group(3)), int(m.group(4))
    for pattern in (r"(\d{4})\s*年\s*(\d{1,2})\s*月\s*(\d{1,2})\s*日", r"(\d{4})[/\-](\d{1,2})[/\-](\d{1,2})"):
        m = re.search(pattern, text)
        if m:
            return int(m.group(1)), int(m.group(2)), int(m.group(3))
    return None


@_rule("date_jp")
def date_jp(text):
    """YYYY-MM-DD, or the text unchanged if no date is found."""
    ymd = _parse_date(text)
    return "%04d-%02d-%02d" % ymd if ymd else text


@_rule("date_yyyymmdd")
def date_yyyymmdd(text):
    """YYYYMMDD, or the text unchanged if no date is found."""
    ymd = _parse_date(text)
    return "%04d%02d%02d" % ymd if ymd else text


def _parse_time(text):
    """(hours, minutes, seconds or None) of the first of 14時30分5秒, 14時30分, 14:30:05, 14:30 found, or None."""
    text = full_to_half(text)
    for pattern in (r"(\d{1,2})\s*時\s*(\d{1,2})\s*分\s*(\d{1,2})\s*秒", r"(\d{1,2})\s*時\s*(\d{1,2})\s*分",
                    r"(\d{1,2})\s*:\s*(\d{1,2})\s*:\s*(\d{1,2})", r"(\d{1,2})\s*:\s*(\d{1,2})"):
        m = re.search(pattern, text)
        if m:
            g = [int(v) for v in m.groups()]
            return g[0], g[1], g[2] if len(g) == 3 else None
    return None


@_rule("time_jp")
def time_jp(text):
    """H時MM分 or H時MM分SS秒, or the text unchanged."""
    t = _parse_time(text)
    if t is None:
        return text
    return "%d時%02d分" % t[:2] + ("%02d秒" % t[2] if t[2] is not None else "")


@_rule("time_hms")
def time_hms(text):
    """HH:MM:SS (seconds 00 when absent), or the text unchanged."""
    t = _parse_time(text)
    if t is None:
        return text
    return "%02d:%02d:%02d" % (t[0], t[1], t[2] or 0)


@_rule("alphanumeric")
def alphanumeric(text):
    return re.sub(r"[^a-zA-Z0-9]", "", full_to_half(text))


@_rule("hiragana")
def hiragana(text):
    """Katakana to hiragana, then only the hiragana block U+3040-U+309F is kept."""
    return re.sub(r"[^\u3040-\u309F]", "", kata_to_hira(text))


@_rule("katakana")
def katakana(text):
    """Hiragana to katakana, then only the katakana block U+30A0-U+30FF is kept (ー stays)."""
    return re.sub(r"[^\u30A0-\u30FF]", "", hira_to_kata(text))


# ------------------------------------------------------------------------------------------------ field extraction
@dataclass
class ResolvedElement:
    id: str
    box: List[Any]
    contents: str
    label: str = ""


@dataclass
class ResolvedField:
    name: str
    value: Any
    raw_text: str
    elements: List[ResolvedElement] = field(default_factory=list)
    confidence: str = "low"
    source: str = "not_found"


def _no_spaces(text):
    return re.sub(r"[ \u3000]", "", text)


def _element(eid, box, contents, label=""):
    return ResolvedElement(id=eid, box=list(box), contents=contents, label=label)


def _one(fs, obj, source, confidence="high", eid=None, value=None):
    """A field resolved to one cell or paragraph: its text, or `value` (a regex match) with the text as raw_text."""
    contents = obj.contents or ""
    return ResolvedField(fs.name, contents if value is None else value, contents,
                         [_element(obj.id if eid is None else eid, obj.box, contents)], confidence, source)


def _by_regex(info, fs):
    pattern = re.compile(fs.regex)
    for table in info.tables:
        for cell in table.cells.values():
            if cell.role != "group" and cell.contents:
                m = pattern.search(cell.contents)
                if m:
                    return _one(fs, cell, "regex", value=m.group(0))
    for i, p in enumerate(info.paragraphs):
        if p.contents:
            m = pattern.search(p.contents)
            if m:
                return _one(fs, p, "regex", eid=p.id or "p%d" % i, value=m.group(0))
    for i, w in enumerate(info.words):
        if w.content:
            m = pattern.search(w.content)
            if m:
                return ResolvedField(fs.name, m.group(0), w.content,
                                     [_element("w%d" % i, quad_to_xyxy(w.points), w.content)], "high", "regex")
    return None


def _by_key(info, fs):
    """Step 3: the value cell(s) of the key-value items whose key text contains the description.  A hit on a grid
    column header (search_kv_items_by_key's grid branch) carries no value cell and is passed over."""
    hits = [r["value"] for r in info.search_kv_items_by_key(fs.description)]
    if fs.merge_values and len(hits) > 1:
        cells = [c for c in hits if c is not None and not isinstance(c, list)]
        if not cells:
            return None
        xs, ys = [c.box[0] for c in cells], [c.box[1] for c in cells]
        axis = 1 if max(ys) - min(ys) >= max(xs) - min(xs) else 0
        cells.sort(key=lambda c: c.box[axis])
        text = fs.separator.join(c.contents or "" for c in cells)
        return ResolvedField(fs.name, text, text, [_element(c.id, c.box, c.contents or "") for c in cells], "high",
                             "kv")
    if hits and hits[0] is not None and not isinstance(hits[0], list):
        return _one(fs, hits[0], "kv")
    return None


def _scalar_field(info, fs):
    if fs.cell_id:
        for table in info.tables:
            cell = table.find_cell_by_id(fs.cell_id)
            if cell is not None:
                return _one(fs, cell, "cell_id")
    if fs.bbox:
        for table in info.tables:
            cells = table.search_cells_by_bbox(fs.bbox)
            if cells:
                return _one(fs, cells[0], "bbox")
    if fs.description:
        found = _by_key(info, fs)
        if found is not None:
            return found
        for table in info.tables:
            cells = table.search_cells_by_query(fs.description)
            if cells:
                return _one(fs, cells[0], "cell_query", "medium")
        q = _no_spaces(fs.description)
        for p in info.paragraphs:
            if p.contents and q in _no_spaces(p.contents):
                return _one(fs, p, "paragraph", "medium", eid=p.id or "p0")
    if fs.regex:
        found = _by_regex(info, fs)
        if found is not None:
            return found
    return ResolvedField(fs.name, "", "", [], "low", "not_found")


def _header_matches(table, header_ids, col):
    if col.cell_id:
        return col.cell_id in header_ids
    if col.bbox:
        return any(table.cells.get(h) is not None and table.cells[h].box and
                   overlap_ratio(col.bbox, list(table.cells[h].box))[0] > 0.5 for h in header_ids)
    text = "".join(table.cells[h].contents or "" for h in header_ids if table.cells.get(h))
    return _no_spaces(col.description or col.name) in _no_spaces(text)


def _table_field(info, fs):
    if not fs.columns:
        return ResolvedField(fs.name, [], "", [], "low", "not_found")
    records, elements = [], []
    for table in info.tables:
        for grid in table.grids:
            columns = {}                                  # schema column name -> grid column indices
            for i, header_ids in enumerate(grid.col_headers):
                col = next((c for c in fs.columns if _header_matches(table, header_ids, c)), None)
                if col is not None:
                    columns.setdefault(col.name, []).append(i)
            if not columns:
                continue
            header_cells = {h for ids in grid.col_headers for h in ids}
            for row in grid.data:
                ids = [c for c in row if c is not None]
                if ids and all(c in header_cells for c in ids):
                    continue
                record = {}
                for name, indices in columns.items():
                    values, cell_ids = [], []
                    for i in indices:
                        cid = row[i] if i < len(row) else None
                        if cid is None:
                            continue
                        cell_ids.append(cid)
                        cell = table.cells.get(cid)
                        if cell:
                            values.append(cell.contents or "")
                            elements.append(_element(cid, cell.box, cell.contents or "", label=name))
                    record[name] = {"value": "".join(values), "cell_ids": cell_ids}
                if record:
                    records.append(record)
    return ResolvedField(fs.name, records, "", elements, "high" if records else "low",
                         "grid" if records else "not_found")


def resolve_fields(semantic_info, schema):
    """One ResolvedField per schema field, in schema order, values not yet normalised."""
    return [_table_field(semantic_info, fs) if fs.structure == "table" else _scalar_field(semantic_info, fs)
            for fs in schema.fields]


def normalize_fields(fields, schema):
    """Applies each field's (each table column's) normalisation rule to its value(s), in place; returns `fields`."""
    by_name = {fs.name: fs for fs in schema.fields}
    for rf in fields:
        fs = by_name.get(rf.name)
        if fs is None:
            continue
        if fs.structure in ("scalar", "kv") and isinstance(rf.value, str):
            rf.value = apply_normalize(rf.value, fs.normalize)
        elif fs.structure == "table" and isinstance(rf.value, list):
            cols = {c.name: c for c in fs.columns or []}
            for row in rf.value:
                if not isinstance(row, dict):
                    continue
                for name, cell in row.items():
                    col = cols.get(name)
                    if col is not None and col.normalize and isinstance(cell, dict):
                        cell["value"] = apply_normalize(cell.get("value", ""), col.normalize)
    return fields


# ------------------------------------------------------------------------------------------------ output
def build_output(fields):
    """{"fields": {name: ...}, "metadata": {"schema_version": "1.0"}}.  A scalar field: structure "kv", value,
    raw_text, confidence, source, cell_ids, bboxes.  A table field: structure "table", records (per column: value,
    cell_ids, raw_text = the cells' texts joined by spaces, bboxes) and source."""
    out = {"fields": {}, "metadata": {"schema_version": SCHEMA_VERSION}}
    for rf in fields:
        if isinstance(rf.value, list):
            boxes = {e.id: e.box for e in rf.elements}
            texts = {e.id: e.contents for e in rf.elements}
            records = []
            for row in rf.value:
                if not isinstance(row, dict):
                    records.append(row)
                    continue
                rec = {}
                for name, cell in row.items():
                    if isinstance(cell, dict):
                        ids = cell.get("cell_ids", [])
                        cell = dict(cell, raw_text=" ".join(texts[c] for c in ids if c in texts),
                                    bboxes=[boxes[c] for c in ids if c in boxes])
                    rec[name] = cell
                records.append(rec)
            out["fields"][rf.name] = {"structure": "table", "records": records, "source": rf.source}
        else:
            out["fields"][rf.name] = {"structure": "kv", "value": rf.value, "raw_text": rf.raw_text,
                                      "confidence": rf.confidence, "source": rf.source,
                                      "cell_ids": [e.id for e in rf.elements], "bboxes": [e.box for e in rf.elements]}
    return out


def build_simple_output(fields):
    """{name: value} for scalar fields, {name: [{column: value}]} for table fields."""
    out = {}
    for rf in fields:
        if isinstance(rf.value, list):
            out[rf.name] = [{k: v.get("value", "") if isinstance(v, dict) else v for k, v in row.items()}
                            if isinstance(row, dict) else row for row in rf.value]
        elif isinstance(rf.value, dict):
            out[rf.name] = rf.value.get("value", "")
        else:
            out[rf.name] = rf.value
    return out


def extract(semantic_info, schema, normalize=True, simple=False):
    """The schema's fields from one TableSemanticParserSchema (what TableSemanticParser returns for a page):
    build_output's form, or {name: value} with simple=True.  `schema`: ExtractionSchema, dict or YAML path."""
    schema = as_schema(schema)
    fields = resolve_fields(semantic_info, schema)
    if normalize:
        normalize_fields(fields, schema)
    return build_simple_output(fields) if simple else build_output(fields)
