"""Writers that turn a `DocumentAnalyzerSchema` into a document: Markdown, HTML, CSV and JSON, with the figures of the
page cut out as image files.  Signatures, defaults and output follow yomitoku's exporters
(src/yomitoku/export/export_{markdown,html,csv,json}.py), so files written by either package are interchangeable:

    convert_markdown / export_markdown / save_markdown
    convert_html     / export_html     / save_html
    convert_csv      / export_csv      / save_csv
    convert_json     / export_json     / save_json

Differences from yomitoku:
  * HTML is written as the element string the exporter builds.  yomitoku re-parses that string with lxml to indent it;
    lxml is not a dependency here, so that indentation (whitespace only) is not reproduced.
  * The caller's result is never modified: `convert_json` works on a deep copy (yomitoku edits its input in place, e.g.
    for `ignore_line_break` and `figure_path`).
  * `export_figure` without `img` raises ValueError (an assertion in yomitoku).

Figures: figure i of `out_path` is `img[y1:y2, x1:x2]` of its int box, written JPEG-encoded (cv2.imencode(".jpg")) to
`<dir of out_path>/<figure_dir>/<stem of out_path>_figure_<i>.png`.  The `.png` name holding JPEG bytes is yomitoku's
and is kept so that links in existing outputs stay valid.  `img` is the BGR page: a numpy array or a CUDA (H, W, 3)
uint8 tensor (a page that never left the device); of a tensor only each figure's rectangle is copied to the host.
"""
import csv
import html
import json
import os
import re

import cv2
import torch


# ------------------------------------------------------------------------------------------------ figures
def _figure_path(out_path, figure_dir, i):
    """(path of figure i's file, its name)."""
    stem = os.path.splitext(os.path.basename(out_path))[0]
    name = "%s_figure_%d.png" % (stem, i)
    return os.path.join(os.path.dirname(out_path), figure_dir, name), name


def _figure_crop(img, box):
    """The figure's rectangle of the page as a host array; of a device page only this rectangle crosses to the host."""
    x1, y1, x2, y2 = map(int, box)
    crop = img[y1:y2, x1:x2, :]
    if torch.is_tensor(crop):
        crop = crop.cpu().numpy()
    return crop


def _write_figure(crop, path):
    ok, buf = cv2.imencode(".jpg", crop)
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    if not ok:
        raise ValueError("Failed to encode image")
    with open(path, "wb") as f:
        f.write(buf.tobytes())


def save_figures(figures, img, out_path, figure_dir="figures"):
    """Writes every figure's crop; returns the file names (relative to the figure directory) in figure order."""
    if img is None:
        raise ValueError("img is required for saving figures")
    names = []
    for i, figure in enumerate(figures):
        path, name = _figure_path(out_path, figure_dir, i)
        _write_figure(_figure_crop(img, figure.box), path)
        names.append(name)
    return names


def _line_breaks(text, ignore_line_break, replacement):
    return text.replace("\n", "" if ignore_line_break else replacement)


def _by_order(elements):
    return sorted(elements, key=lambda e: e["order"])


def _write_text(text, out_path, encoding):
    with open(out_path, "w", encoding=encoding, errors="ignore") as f:
        f.write(text)


# ------------------------------------------------------------------------------------------------ Markdown
_MD_SPECIAL = set("`*{}[]()#+!~|-")


def escape_markdown_special_chars(text):
    """A backslash before each Markdown special character: ` * { } [ ] ( ) # + ! ~ | -"""
    return "".join("\\" + c if c in _MD_SPECIAL else c for c in text)


def paragraph_to_md(paragraph, ignore_line_break):
    md = _line_breaks(escape_markdown_special_chars(paragraph.contents), ignore_line_break, "<br>")
    if paragraph.role == "section_headings":
        md = "# " + md
    return {"order": paragraph.order, "box": paragraph.box, "md": md + "\n"}


def table_to_md(table, ignore_line_break):
    """n_row x n_col pipe grid; a spanned cell's text sits in its top-left slot, a |-|...| rule follows row 1."""
    grid = [[""] * table.n_col for _ in range(table.n_row)]
    for cell in table.cells:
        if cell.row_span > 0 and cell.col_span > 0:
            text = _line_breaks(escape_markdown_special_chars(cell.contents), ignore_line_break, "<br>")
            grid[cell.row - 1][cell.col - 1] = text
    lines = []
    for i, row in enumerate(grid):
        lines.append("|%s|\n" % "|".join(row))
        if i == 0:
            lines.append("|%s|\n" % "|".join(["-"] * table.n_col))
    return {"order": table.order, "box": table.box, "md": "".join(lines)}


def figure_to_md(figures, img, out_path, export_figure_letter=False, ignore_line_break=False, width=200,
                 figure_dir="figures"):
    elements = []
    for figure, name in zip(figures, save_figures(figures, img, out_path, figure_dir)):
        elements.append({"order": figure.order,
                         "md": '<img src="%s/%s" width="%spx"><br>' % (figure_dir, name, width)})
        if export_figure_letter:
            for p in sorted(figure.paragraphs, key=lambda p: p.order):
                elements.append({"order": figure.order, "md": paragraph_to_md(p, ignore_line_break)["md"]})
    return elements


def convert_markdown(inputs, out_path, ignore_line_break=False, img=None, export_figure_letter=False,
                     export_figure=True, figure_width=200, figure_dir="figures"):
    """(markdown string, its elements): tables, paragraphs and (with export_figure) figures sorted by order, joined by
    newlines."""
    elements = [table_to_md(t, ignore_line_break) for t in inputs.tables]
    elements += [paragraph_to_md(p, ignore_line_break) for p in inputs.paragraphs]
    if export_figure:
        elements += figure_to_md(inputs.figures, img, out_path, export_figure_letter, ignore_line_break, figure_width,
                                 figure_dir=figure_dir)
    elements = _by_order(elements)
    return "\n".join(e["md"] for e in elements), elements


def export_markdown(inputs, out_path: str, ignore_line_break: bool = False, img=None, export_figure_letter=False,
                    export_figure=True, figure_width=200, figure_dir="figures", encoding: str = "utf-8"):
    markdown, _ = convert_markdown(inputs, out_path, ignore_line_break, img, export_figure_letter, export_figure,
                                   figure_width, figure_dir)
    save_markdown(markdown, out_path, encoding)
    return markdown


def save_markdown(markdown, out_path, encoding):
    _write_text(markdown, out_path, encoding)


# ------------------------------------------------------------------------------------------------ HTML
_URL_HEAD = re.compile(r"https?://[^\s<>]")


def convert_text_to_html(text):
    """html.escape(text), after which each "http(s)://" plus the character that follows it is escaped once more, as
    yomitoku does: "&" right after "://" (from an escaped &, <, >, " or ') ends up as "&amp;amp;"."""
    return _URL_HEAD.sub(lambda m: html.escape(m.group(0)), html.escape(text))


def table_to_html(table, ignore_line_break):
    """One <tr> per run of cells with the same `row`, one <td rowspan colspan> per cell (None contents -> "")."""
    rows, row, prev = [], [], 1
    for cell in table.cells:
        if cell.row != prev:
            rows.append(row)
            row = []
        text = _line_breaks(convert_text_to_html(cell.contents or ""), ignore_line_break, "<br>")
        row.append('<td rowspan="%s" colspan="%s">%s</td>' % (cell.row_span, cell.col_span, text))
        prev = cell.row
    rows.append(row)
    body = "".join("<tr>%s</tr>" % "".join(r) for r in rows)
    return {"box": table.box, "order": table.order,
            "html": '<table border="1" style="border-collapse: collapse">%s</table>' % body}


def paragraph_to_html(paragraph, ignore_line_break):
    text = _line_breaks(convert_text_to_html(paragraph.contents), ignore_line_break, "<br>")
    if paragraph.role == "section_headings":
        text = "<h1>%s</h1>" % text
    return {"box": paragraph.box, "order": paragraph.order, "html": "<p>%s</p>" % text}


def figure_to_html(figures, img, out_path, export_figure_letter=False, ignore_line_break=False, figure_dir="figures",
                   width=200):
    elements = []
    for figure, name in zip(figures, save_figures(figures, img, out_path, figure_dir)):
        elements.append({"order": figure.order,
                         "html": '<img src="%s/%s" width="%s"><br>' % (figure_dir, name, width)})
        if export_figure_letter:
            for p in sorted(figure.paragraphs, key=lambda p: p.order):
                elements.append({"order": figure.order, "html": paragraph_to_html(p, ignore_line_break)["html"]})
    return elements


def convert_html(inputs, out_path, ignore_line_break, export_figure, export_figure_letter, img=None, figure_width=200,
                 figure_dir="figures"):
    """(HTML string, its elements): the elements sorted by order and concatenated.  yomitoku re-indents this string
    with lxml; here it is returned as built (see the module docstring)."""
    elements = [table_to_html(t, ignore_line_break) for t in inputs.tables]
    elements += [paragraph_to_html(p, ignore_line_break) for p in inputs.paragraphs]
    if export_figure:
        elements += figure_to_html(inputs.figures, img, out_path, export_figure_letter, ignore_line_break,
                                   width=figure_width, figure_dir=figure_dir)
    elements = _by_order(elements)
    return "".join(e["html"] for e in elements), elements


def export_html(inputs, out_path: str, ignore_line_break: bool = False, export_figure: bool = True,
                export_figure_letter: bool = False, img=None, figure_width=200, figure_dir="figures",
                encoding: str = "utf-8"):
    text, _ = convert_html(inputs, out_path, ignore_line_break, export_figure, export_figure_letter, img, figure_width,
                           figure_dir)
    save_html(text, out_path, encoding)
    return text


def save_html(html_string, out_path, encoding):
    _write_text(html_string, out_path, encoding)


# ------------------------------------------------------------------------------------------------ CSV
def table_to_csv(table, ignore_line_break):
    """n_row x n_col rows; a spanned cell's text sits in its top-left slot."""
    grid = [[""] * table.n_col for _ in range(table.n_row)]
    for cell in table.cells:
        text = cell.contents.replace("\n", "") if ignore_line_break else cell.contents
        if cell.row_span > 0 and cell.col_span > 0:
            grid[cell.row - 1][cell.col - 1] = text
    return grid


def paragraph_to_csv(paragraph, ignore_line_break):
    return paragraph.contents.replace("\n", "") if ignore_line_break else paragraph.contents


def convert_csv(inputs, out_path, ignore_line_break, img=None, export_figure: bool = True,
                export_figure_letter: bool = False, figure_dir="figures"):
    """The elements to write, sorted by order: tables (rows), paragraphs and, with export_figure_letter, each figure's
    paragraphs in the figure's place.  With export_figure the figure crops are written."""
    elements = [{"type": "table", "box": t.box, "element": table_to_csv(t, ignore_line_break), "order": t.order}
                for t in inputs.tables]
    elements += [{"type": "paragraph", "box": p.box, "element": paragraph_to_csv(p, ignore_line_break),
                  "order": p.order} for p in inputs.paragraphs]
    if export_figure_letter:
        for figure in inputs.figures:
            for p in sorted(figure.paragraphs, key=lambda p: p.order):
                elements.append({"type": "paragraph", "box": p.box, "element": paragraph_to_csv(p, ignore_line_break),
                                 "order": figure.order})
    elements = _by_order(elements)
    if export_figure:
        save_figures(inputs.figures, img, out_path, figure_dir)
    return elements


def export_csv(inputs, out_path: str, ignore_line_break: bool = False, encoding: str = "utf-8", img=None,
               export_figure: bool = True, export_figure_letter: bool = False, figure_dir="figures"):
    elements = convert_csv(inputs, out_path, ignore_line_break, img, export_figure, export_figure_letter, figure_dir)
    save_csv(elements, out_path, encoding)
    return elements


def save_csv(elements, out_path, encoding):
    """A table as its rows, a paragraph as one row; every element is followed by the row [""]."""
    with open(out_path, "w", newline="", encoding=encoding, errors="ignore") as f:
        writer = csv.writer(f, quoting=csv.QUOTE_MINIMAL)
        for e in elements:
            if e["type"] == "table":
                writer.writerows(e["element"])
            else:
                writer.writerow([e["element"]])
            writer.writerow([""])


# ------------------------------------------------------------------------------------------------ JSON
def convert_json(inputs, out_path, ignore_line_break, img, export_figure, figure_dir):
    """A deep copy of `inputs`; for a DocumentAnalyzerSchema with ignore_line_break applied to paragraph and cell
    contents, and with export_figure each figure written and its `figure_path` (relative to out_path's directory)
    set."""
    from .schemas import DocumentAnalyzerSchema
    out = inputs.model_copy(deep=True)
    if not isinstance(out, DocumentAnalyzerSchema):
        return out
    if ignore_line_break:
        for table in out.tables:
            for cell in table.cells:
                cell.contents = cell.contents.replace("\n", "")
        for p in out.paragraphs:
            p.contents = p.contents.replace("\n", "")
    if export_figure:
        for figure, name in zip(out.figures, save_figures(out.figures, img, out_path, figure_dir)):
            figure.figure_path = os.path.join(figure_dir, name)
    return out


def export_json(inputs, out_path, ignore_line_break=False, encoding: str = "utf-8", img=None, export_figure=False,
                figure_dir="figures"):
    """Writes `model_dump()` as yomitoku's exporter does (4-space indent, sorted keys, non-ASCII kept) and returns the
    exported copy of `inputs`."""
    out = convert_json(inputs, out_path, ignore_line_break, img, export_figure, figure_dir)
    save_json(out.model_dump(), out_path, encoding)
    return out


def save_json(data, out_path, encoding):
    with open(out_path, "w", encoding=encoding, errors="ignore") as f:
        json.dump(data, f, ensure_ascii=False, indent=4, sort_keys=True, separators=(",", ": "))
