"""Result types of the hot path (pydantic), mirroring reference src/yomitoku/schemas/document_analyzer.py:137-180,
234-254, schemas/table_semantic_parser.py and BaseSchema (base.py:51-57): extra fields forbidden, assignment
validated."""
import json
import os
import re
from collections import defaultdict
from typing import Any, Dict, List, Literal, Optional, Union

from pydantic import BaseModel, ConfigDict, Field, conlist

Quad = conlist(conlist(int, min_length=2, max_length=2), min_length=4, max_length=4)


class BaseSchema(BaseModel):
    model_config = ConfigDict(extra="forbid", validate_assignment=True)

    def to_json(self, out_path: str, **kwargs):
        import json
        with open(out_path, "w", encoding="utf-8") as f:
            json.dump(self.model_dump(), f, ensure_ascii=False, indent=kwargs.get("indent", 4))


class WordPrediction(BaseSchema):
    points: Quad = Field(..., description="[[x1, y1], [x2, y2], [x3, y3], [x4, y4]]")
    content: str = Field(..., description="Text content of the word")
    direction: str = Field(..., description="'horizontal' or 'vertical'")
    rec_score: float = Field(..., description="Confidence score of the word recognition")
    det_score: float = Field(..., description="Confidence score of the word detection")


class TextDetectorSchema(BaseSchema):
    points: List[Quad] = Field(..., description="Detected text regions as quadrilaterals")
    scores: List[float] = Field(..., description="Confidence score per region")


class TextRecognizerSchema(BaseSchema):
    contents: List[str] = Field(..., description="Recognized text contents")
    directions: List[str] = Field(..., description="'horizontal' or 'vertical' per text")
    scores: List[float] = Field(..., description="Confidence score per text")
    points: List[Quad] = Field(..., description="Quadrilaterals of the recognized texts")


class OCRSchema(BaseSchema):
    words: List[WordPrediction] = Field(..., description="Recognized words")


Box = conlist(int, min_length=4, max_length=4)


class Element(BaseSchema):
    """One layout region (reference schemas/document_analyzer.py:9-29): what a layout analyzer returns per paragraph /
    figure."""
    id: Union[str, None] = Field(None, description="Unique identifier of the element")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    score: float = Field(..., description="Detection confidence")
    role: Union[str, None] = Field(..., description="e.g. 'section_headings', 'page_header', 'page_footer'")
    contents: Union[str, None] = Field(None, description="Text content of the element")


class ParagraphSchema(BaseSchema):
    box: Box
    contents: Union[str, None]
    direction: Union[str, None]
    order: Union[int, None]
    role: Union[str, None]


class TableCellSchema(BaseSchema):
    col: int
    row: int
    col_span: int
    row_span: int
    box: Box
    contents: Union[str, None]


class TableLineSchema(BaseSchema):
    box: Box
    score: float


class TableStructureRecognizerSchema(BaseSchema):
    """reference schemas/document_analyzer.py:94-118."""
    box: Box
    n_row: int
    n_col: int
    rows: List[TableLineSchema]
    cols: List[TableLineSchema]
    spans: List[TableLineSchema] = Field(default_factory=list)
    cells: List[TableCellSchema]
    order: int


class LayoutParserSchema(BaseSchema):
    """reference schemas/document_analyzer.py:183-186: what LayoutParser returns (tables are plain regions here)."""
    paragraphs: List[Element]
    tables: List[Element]
    figures: List[Element]


class LayoutAnalyzerSchema(BaseSchema):
    """What the layout half (reference layout_analyzer.py:38-49) hands to DocumentAnalyzer.aggregate."""
    paragraphs: List[Element]
    tables: List[TableStructureRecognizerSchema]
    figures: List[Element]


class FigureSchema(BaseSchema):
    box: Box
    order: Union[int, None]
    paragraphs: List[ParagraphSchema]
    direction: Union[str, None]
    figure_path: Union[str, None] = None


class DocumentAnalyzerSchema(BaseSchema):
    """reference DocumentAnalyzerSchema (schemas/document_analyzer.py:207-226).  Tables / figures / layout paragraphs
    come from a layout analyzer (the RT-DETRv2 models are outside this repo's hot path, SURVEY.md section 8f); without
    one every word becomes its own paragraph, exactly what the reference's aggregate does with an empty layout."""
    paragraphs: List[ParagraphSchema] = Field(default_factory=list)
    tables: List[TableStructureRecognizerSchema] = Field(default_factory=list)
    words: List[WordPrediction] = Field(default_factory=list)
    figures: List[FigureSchema] = Field(default_factory=list)


# ------------------------------------------------------------------------------------------------ cell detector
class CellSchema(BaseSchema):
    """One cell of a table crop (reference schemas/table_semantic_parser.py:62-101); row / col / spans stay None until a
    table parser assigns them."""
    meta: Dict[str, Any] = Field(default_factory=dict, description="Additional metadata for template/semantics")
    contents: Union[str, None] = Field(..., description="Text content of the cell")
    role: Union[str, None] = Field(..., description="'cell', 'header', 'empty' or 'group'")
    id: Union[str, None] = Field(..., description="Unique identifier of the cell")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    row: Union[int, None] = Field(..., description="Row index of the cell in the table")
    col: Union[int, None] = Field(..., description="Column index of the cell in the table")
    row_span: Union[int, None] = Field(..., description="Number of rows spanned by the cell")
    col_span: Union[int, None] = Field(..., description="Number of columns spanned by the cell")


class RegionSchema(BaseSchema):
    """A kv_item / grid region as the model predicts it (reference schemas/table_semantic_parser.py:104-112)."""
    id: Union[str, None] = Field(None, description="Region id")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    role: str = Field(..., description="'kv_item' or 'grid'")
    score: float = Field(1.0, description="Detection score")


class TableDetectorSchema(BaseSchema):
    """What CellDetector returns per table (reference schemas/table_semantic_parser.py:115-140)."""
    id: Union[str, None] = Field(..., description="Unique identifier of the table")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    role: Union[str, None] = Field(..., description="Role of the table region")
    cells: List[CellSchema] = Field(..., description="List of detected table cells")
    kv_regions: List[RegionSchema] = Field(default_factory=list, description="Model-predicted key-value item regions")
    grid_regions: List[RegionSchema] = Field(default_factory=list, description="Model-predicted grid regions")


# ------------------------------------------------------------------------------------------------ table semantic parser
class KvItemSchema(BaseSchema):
    """One key-value item: the key cell ids (outermost header first) and the value cell id (reference
    schemas/table_semantic_parser.py:143-153)."""
    id: Union[str, None] = Field(..., description="Unique identifier of the key-value item")
    key: Union[str, List[str]] = Field(..., description="Key cell id(s)")
    value: str = Field(..., description="Value cell id")
    box: Union[Box, None] = Field(None, description="[x1, y1, x2, y2] of the key and the value")


class TableGridSchema(BaseSchema):
    """One grid: cell ids per row and column (None where no cell is), column header ids per column (:156-180)."""
    id: Union[str, None] = Field(..., description="Unique identifier of the table grid")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    n_row: int = Field(..., description="Number of rows in the table grid")
    n_col: int = Field(..., description="Number of columns in the table grid")
    col_headers: List[List[str]] = Field(..., description="Column header cell ids per column")
    data: List[List[Union[str, None]]] = Field(..., description="Cell ids of the grid, row by row")


def _strip_spaces(text):
    """Without half- and full-width spaces (reference :49-51)."""
    return re.sub(r"[ 　]", "", text)


def _numbered_duplicates(keys):
    """Each key (a list) that occurs more than once gets its occurrence number appended (reference :32-46)."""
    counts = defaultdict(int)
    out = []
    for k in keys:
        out.append(k + [counts[tuple(k)]])
        counts[tuple(k)] += 1
    for o, k in zip(out, keys):
        if counts[tuple(k)] == 1:
            o.pop()
    return out


class TableSemanticContentsSchema(BaseSchema):
    """One table: its cells by id, key-value items and grids (reference :299-518, the export / view helpers it needs
    for `to_dict` and `to_csv`: :539-569, 613-646, 662-706, 729-783)."""
    id: Union[str, None] = Field(None, description="Unique identifier of the table")
    style: str = Field(..., description="Border style of the table, e.g. 'border', 'borderless'")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    cells: Dict[str, CellSchema] = Field(..., description="Cells keyed by cell id")
    kv_items: List[KvItemSchema] = Field(..., description="Key-value items extracted from the table")
    grids: List[TableGridSchema] = Field(..., description="Grid representation of the table")

    def safe_contents(self, cell_id, ignore_space=True):
        """The cell's text ("" for an unknown id or no text), without half-width spaces unless ignore_space=False."""
        c = self.cells.get(cell_id)
        contents = (c.contents or "") if c is not None else ""
        return contents.replace(" ", "") if ignore_space else contents

    def find_cell_by_id(self, cell_id):
        return self.cells.get(str(cell_id))

    def search_cells_by_bbox(self, box):
        """Non-group cells more than half inside box."""
        from .document_analyzer import is_contained
        return [c for c in self.cells.values() if c.role != "group" and is_contained(box, c.box, threshold=0.5)]

    def search_kv_items_by_key(self, key):
        """[{"key": key cells, "value": value cell}] of the items whose key text contains `key` (spaces ignored), then
        for every grid column whose header text contains it one {"key": header cells, "value": []} per grid row - the
        reference's grid branch (:444-457) looks the header text up by contents instead of id and never fills the
        value list; kept as it is."""
        q = _strip_spaces(key)
        results = []
        for kv in self.kv_items:
            key_cells = [self.cells.get(k) for k in kv.key]
            if q in _strip_spaces("".join((kc.contents or "") for kc in key_cells if kc)):
                results.append({"key": key_cells, "value": self.cells.get(kv.value)})
        for grid in self.grids:
            for col in grid.col_headers:
                col_cells = [self.cells.get(ck) for ck in col]
                if q in _strip_spaces("".join(self.safe_contents(c.contents) for c in col_cells if c)):
                    results.extend({"key": col_cells, "value": []} for _ in grid.data)
        return results

    def find_table_by_column_name(self, queries):
        """This table with every grid reduced to the columns whose header text contains one of `queries`."""
        grids = [g for g in (self.filter_columns_ignore_space(grid, queries) for grid in self.grids) if g is not None]
        return TableSemanticContentsSchema(id=self.id, box=self.box, style=self.style, cells=self.cells, grids=grids,
                                           kv_items=self.kv_items)

    def filter_columns_ignore_space(self, grid, queries):
        queries = [_strip_spaces(q) for q in queries]
        data, n_col, headers = [], None, defaultdict(int)
        for row in grid.data:
            kept = []
            for i, cell in enumerate(row):
                nk = _strip_spaces("".join(self.cells.get(rk).contents or "" for rk in grid.col_headers[i]))
                if any(q in nk for q in queries):
                    kept.append(cell)
                    headers[tuple(grid.col_headers[i])] += 1
            if kept:
                data.append(kept)
                n_col = len(kept)
        if not data:
            return None
        return TableGridSchema(id=grid.id, data=data, n_col=n_col, n_row=len(data), col_headers=list(headers.keys()),
                               box=grid.box)

    def grids_to_csv(self, out_path, columns=None, ignore_space=True):
        """Writes each grid as `<out_path without extension>_<grid id>.csv` (cell texts joined by commas) and returns
        the rows; `columns` keeps only the columns whose header text contains one of them."""
        table = self.find_table_by_column_name(queries=columns) if columns is not None else self
        dirname = os.path.dirname(out_path)
        if dirname:
            os.makedirs(dirname, exist_ok=True)
        base = out_path.rsplit(".", 1)[0]
        csvs = []
        for grid in table.grids:
            csv = [[table.safe_contents(cid, ignore_space) for cid in row] for row in grid.data]
            with open("%s_%s.csv" % (base, grid.id), "w", encoding="utf-8") as f:
                for row in csv:
                    f.write(",".join(row) + "\n")
            csvs.append(csv)
        return csvs

    def grids_to_dict(self, ignore_space=True):
        """Per grid {"id", "rows"}: every non-header row as {column header texts joined by "_" (numbered where they
        repeat): cell text}, each cell once."""
        results = []
        for grid in self.grids:
            rows = []
            for row in grid.data:
                seen, keys, values = set(), [], []
                for i, cell in enumerate(row):
                    if cell in grid.col_headers[i] or cell in seen:
                        continue
                    keys.append([self.safe_contents(h, ignore_space) for h in grid.col_headers[i]])
                    values.append(self.safe_contents(cell, ignore_space))
                    seen.add(cell)
                parsed = {"_".join(map(str, k)): v for k, v in zip(_numbered_duplicates(keys), values)}
                if parsed:
                    rows.append(parsed)
            results.append({"id": grid.id, "rows": rows})
        return results

    def _kv_groups(self):
        """Items grouped by their key cell ids (key-less items stay single), values of a group in reading order along
        the axis they spread most."""
        groups, by_key = [], {}
        for kv in self.kv_items:
            key_ids = [kv.key] if isinstance(kv.key, str) else list(kv.key)
            gid = tuple(key_ids)
            if key_ids and gid in by_key:
                group = by_key[gid]
            else:
                group = {"key_ids": list(key_ids), "values": []}
                groups.append(group)
                if key_ids:
                    by_key[gid] = group
            group["values"].append((self.safe_contents(kv.value), self.find_cell_by_id(kv.value)))
        for group in groups:
            values = group["values"]
            if len(values) > 1:
                with_cell = [v for v in values if v[1] is not None]
                if with_cell:
                    boxes = [v[1].box for v in with_cell]
                    spread_x = max(b[0] for b in boxes) - min(b[0] for b in boxes)
                    spread_y = max(b[1] for b in boxes) - min(b[1] for b in boxes)
                    axis = 1 if spread_y >= spread_x else 0
                    with_cell.sort(key=lambda v: v[1].box[axis])
                group["values"] = with_cell + [v for v in values if v[1] is None]
        return groups

    def kv_items_to_nested(self, separator="\n"):
        """The items as a dict nested along their key chains (node identity by cell id; same-text siblings become a
        list; a key with both a value and children keeps the value under "_value"; key-less values under
        "_unkeyed")."""
        root = {"text": None, "children": {}, "order": [], "values": []}
        for i, group in enumerate(self._kv_groups()):
            chain = ([(cid, self.safe_contents(cid)) for cid in group["key_ids"]] if group["key_ids"]
                     else [("__keyless_%d" % i, "_unkeyed")])
            node = root
            for cid, text in chain:
                child = node["children"].get(cid)
                if child is None:
                    child = {"text": text, "children": {}, "order": [], "values": []}
                    node["children"][cid] = child
                    node["order"].append(cid)
                node = child
            node["values"].append(separator.join(str(v[0]) for v in group["values"]))
        return _render_nested(root)


def _render_nested(node):
    by_text = {}
    for cid in node["order"]:
        child = node["children"][cid]
        sub = _render_nested(child)
        if child["values"]:
            sub = {"_value": child["values"][0], **sub} if sub else child["values"][0]
        by_text.setdefault(child["text"], []).append(sub)
    return {text: items[0] if len(items) == 1 else items for text, items in by_text.items()}


class TemplateMetaSchema(BaseSchema):
    template_version: str = Field("beta", description="Template schema version")
    template_id: Union[str, None] = Field(None, description="Human-readable template id")
    notes: Union[str, None] = Field(None, description="Notes for template editors")
    match_policy: Literal["cell_id", "bbox"] = Field("cell_id", description="How to match cells")


class CellTemplateSchema(BaseSchema):
    id: Optional[str] = Field(None, description="Cell id for matching")
    box: Optional[Box] = Field(None, description="Cell bbox for matching")
    role: Optional[str] = Field(None, description="Role override")
    contents: Optional[str] = Field(None, description="Contents override")


class TableSemanticContentsTemplateSchema(BaseSchema):
    id: Optional[str] = Field(None, description="Unique identifier of the table (optional)")
    style: Optional[str] = Field(None, description="Border style (optional)")
    box: Box = Field(..., description="[x1, y1, x2, y2]")
    cells: Dict[str, CellTemplateSchema] = Field(default_factory=dict, description="Template cells by id")
    kv_items: Optional[List[KvItemSchema]] = Field(None, description="Optional KV items override")
    grids: Optional[List[TableGridSchema]] = Field(None, description="Optional grids override")


class TableSemanticParserTemplateSchema(BaseSchema):
    """A saved parse that corrects later ones (reference :840-889): per table matched by position, cell roles and
    texts (matched by id or box) and optionally the kv items and grids."""
    meta: TemplateMetaSchema = Field(..., description="Template metadata")
    tables: List[TableSemanticContentsTemplateSchema] = Field(..., description="Template tables")

    def find_table_by_id(self, table_id):
        for table in self.tables:
            if table.id == str(table_id):
                return table


class TableSemanticParserSchema(BaseSchema):
    """What TableSemanticParser returns per page (reference :892-1097)."""
    tables: List[TableSemanticContentsSchema] = Field(..., description="Tables with semantic information")
    paragraphs: List[Element] = Field(..., description="Recognized paragraphs of the page")
    words: List[WordPrediction] = Field(..., description="Recognized words of the page")

    @classmethod
    def load_json(cls, json_path):
        with open(json_path, "r", encoding="utf-8") as f:
            return cls.model_validate(json.load(f))

    def to_csv(self, outdir):
        for table in self.tables:
            table.grids_to_csv(out_path="%s/table_%s.csv" % (outdir, table.id))

    def to_dict(self, separator="\n"):
        """table id -> {"kv_items": nested key-value dict, "grids": rows as {column header: text}}."""
        return {t.id: {"kv_items": t.kv_items_to_nested(separator=separator), "grids": t.grids_to_dict()}
                for t in self.tables}

    def find_table_by_id(self, table_id):
        for table in self.tables:
            if table.id == str(table_id):
                return table

    def find_table_by_position(self, box):
        """The table that holds most of box, if more than half of it."""
        from .document_analyzer import overlap_ratio
        ratios = [overlap_ratio(box, t.box)[0] for t in self.tables]
        if not ratios:
            return None
        i = ratios.index(max(ratios))
        return self.tables[i] if ratios[i] > 0.5 else None

    def search_kv_items_by_key(self, key):
        return [r for table in self.tables for r in table.search_kv_items_by_key(key)]

    def load_template_json(self, template_path):
        """Applies a template written by save_template_json (or edited by hand) to this result, in place."""
        with open(template_path, "r", encoding="utf-8") as f:
            template = TableSemanticParserTemplateSchema.model_validate(json.load(f))
        policy = template.meta.match_policy
        for tt in template.tables:
            table = self.find_table_by_position(tt.box)
            if table is None:
                continue
            for tcell in tt.cells.values():
                if policy == "cell_id":
                    cell = table.cells.get(str(tcell.id)) if tcell.id else None
                else:
                    found = table.search_cells_by_bbox(list(tcell.box)) if tcell.box else []
                    cell = found[0] if found else None
                if cell is None:
                    continue
                if tcell.role is not None:
                    cell.role = tcell.role
                if tcell.contents is not None:
                    cell.contents = tcell.contents
            if tt.kv_items is not None:
                table.kv_items = tt.kv_items
            if tt.grids is not None:
                table.grids = tt.grids
        return self

    def save_template_json(self, out_path, include_kv=True, include_grids=True):
        tables = []
        for t in self.tables:
            cells = {str(cid): CellTemplateSchema(id=str(c.id) if c.id is not None else str(cid), box=list(c.box),
                                                  role=c.role, contents=c.contents)
                     for cid, c in t.cells.items() if c.role != "group"}
            tables.append(TableSemanticContentsTemplateSchema(id=t.id, style=t.style, box=list(t.box), cells=cells,
                                                              kv_items=t.kv_items if include_kv else None,
                                                              grids=t.grids if include_grids else None))
        template = TableSemanticParserTemplateSchema(meta=TemplateMetaSchema(), tables=tables)
        with open(out_path, "w", encoding="utf-8") as f:
            json.dump(template.model_dump(exclude_none=True), f, ensure_ascii=False, indent=4)
