"""Command line: `python -m yomitoku_b200 <file-or-dir> -f md -o results`.

Options, defaults and output file names follow yomitoku's `yomitoku` command (src/yomitoku/cli/main.py); what differs
is how the pages run.  The pages of all input files go through `DocumentAnalyzer.analyze_pages` in batches of `--batch`
pages (of any mix of sizes), while one thread decodes the next batch; each batch's outputs are written as soon as it
is done.  Each page's files are what the exporter writes for `analyzer(page)` on that page alone.

    <outdir>/<dir>_<stem>_p<N>.<fmt>      one file per page (N counts from 1)
    <outdir>/<dir>_<stem>.<fmt>           one file per input with --combine
    <outdir>/<figure_dir>/<dir>_<stem>_p<N>_figure_<i>.png    with --figure

<dir> is the input's parent folder name with leading dots replaced by "_".  A file in a directory that cannot be read
as a page image is logged and skipped.

Not available here: the visualisations (-v), searchable-PDF output (-f pdf, --font_path, --pdf_quality) and PDF input
(--dpi): there is no visualiser for the batched path and no PDF renderer among the dependencies.  Searchable PDFs are
written from Python with `create_searchable_pdf(pages, results, path, image_quality=...)` (searchable_pdf.py).
"""
import argparse
import os
import re
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

from . import export
from .base import set_logger
from .data import load_image

logger = set_logger(__name__, "INFO")

SUPPORT_OUTPUT_FORMAT = ["json", "csv", "html", "markdown", "md"]
SUPPORT_ENCODING = ["utf-8", "utf-8-sig", "shift-jis", "euc-jp", "cp932"]


def build_parser():
    p = argparse.ArgumentParser(prog="python -m yomitoku_b200",
                                description="Document analysis of page images into JSON, CSV, HTML or Markdown files.")
    p.add_argument("arg1", type=str, help="path of target image file or directory (searched recursively)")
    p.add_argument("-f", "--format", type=str, default="json", help="output format type (json or csv or html or md)")
    p.add_argument("-o", "--outdir", type=str, default="results", help="output directory")
    p.add_argument("-l", "--lite", action="store_true", help="if set, use lite model (parseq-tiny-dynw-v4)")
    p.add_argument("-d", "--device", type=str, default="cuda", help="device to use")
    p.add_argument("--td_cfg", type=str, default=None, help="path of text detector config file")
    p.add_argument("--tr_cfg", type=str, default=None, help="path of text recognizer config file")
    p.add_argument("--lp_cfg", type=str, default=None, help="path of layout parser config file")
    p.add_argument("--tsr_cfg", type=str, default=None, help="path of table structure recognizer config file")
    p.add_argument("--tr_name", type=str, default="parseq-large-v4_1",
                   help="name of text recognizer model (default: parseq-large-v4_1)")
    p.add_argument("--td_name", type=str, default="dbnetv2_1", help="name of text detector model (default: dbnetv2_1)")
    p.add_argument("--ignore_line_break", action="store_true", help="if set, ignore line break in the output")
    p.add_argument("--figure", action="store_true", help="if set, export figure in the output")
    p.add_argument("--figure_letter", action="store_true", help="if set, export letter within figure in the output")
    p.add_argument("--figure_width", type=int, default=200, help="width of figure image in the output")
    p.add_argument("--figure_dir", type=str, default="figures", help="directory to save figure images")
    p.add_argument("--encoding", type=str, default="utf-8",
                   help="character encoding of the output files (%s); characters it cannot represent are dropped"
                   % ", ".join(SUPPORT_ENCODING))
    p.add_argument("--combine", action="store_true", help="if set, merge all pages of a file in one output")
    p.add_argument("--ignore_meta", action="store_true",
                   help="if set, ignore meta information (header, footer) in the output")
    p.add_argument("--reading_order", default="auto", type=str,
                   choices=["auto", "left2right", "top2bottom", "right2left"])
    p.add_argument("--pages", type=str, default=None,
                   help="pages to process, e.g., 1,2,5-10 (default: all pages, starting from 1)")
    p.add_argument("--enable-rec-orientation-fallback", action="store_true",
                   help="if set, enable orientation fallback for recognition")
    p.add_argument("--rec-orientation-fallback-thresh", type=float, default=0.75,
                   help="confidence threshold for orientation fallback (default: 0.75)")
    p.add_argument("--ignore_ruby", action="store_true", help="if set, ignore ruby (furigana) text in the output")
    p.add_argument("--ruby_threshold", type=float, default=1.0,
                   help="bimodality separation threshold for ruby detection (default: 1.0)")
    p.add_argument("--batch", type=int, default=16, help="pages per analyze_pages call (default: 16)")
    return p


def output_format(args):
    """The validated output format ("markdown" -> "md"); also checks --encoding and --batch."""
    fmt = args.format.lower()
    if fmt == "pdf":
        raise ValueError("Searchable PDF output (-f pdf) is not available on this command line: write it from Python "
                         "with yomitoku_b200.create_searchable_pdf(pages, results, path). Supported formats are %s"
                         % SUPPORT_OUTPUT_FORMAT)
    if fmt not in SUPPORT_OUTPUT_FORMAT:
        raise ValueError(f"Invalid output format: {args.format}. Supported formats are {SUPPORT_OUTPUT_FORMAT}")
    if args.encoding not in SUPPORT_ENCODING:
        raise ValueError(f"Invalid encoding: {args.encoding}")
    if args.batch < 1:
        raise ValueError(f"--batch must be at least 1, got {args.batch}")
    return "md" if fmt == "markdown" else fmt


def parse_pages(pages_str):
    """"1,2,5-10" -> [1, 2, 5, 6, 7, 8, 9, 10]."""
    pages = set()
    for part in pages_str.split(","):
        if "-" in part:
            start, end = map(int, part.split("-"))
            pages.update(range(start, end + 1))
        else:
            pages.add(int(part))
    return sorted(pages)


def _sanitize_path_component(component):
    """Leading dots become underscores, one for one (".scans" -> "_scans")."""
    return re.sub(r"^\.+", lambda m: "_" * len(m.group(0)), component) if component else component


def input_files(path):
    path = Path(path)
    if path.is_dir():
        return sorted(f for f in path.rglob("*") if f.is_file())
    return [path]


def merge_all_pages(fmt, data):
    """One file's pages in one output: JSON as a list, CSV elements concatenated, HTML / Markdown joined by "\\n"."""
    if fmt == "json":
        return list(data)
    if fmt == "csv":
        return [e for page in data for e in page]
    return "\n".join(data)


def save_merged(fmt, out, out_path, encoding):
    save = {"json": export.save_json, "csv": export.save_csv, "html": export.save_html, "md": export.save_markdown}
    save[fmt](out, out_path, encoding)


class _Page:
    __slots__ = ("file", "index", "img", "last")

    def __init__(self, file, index, img, last):
        self.file, self.index, self.img, self.last = file, index, img, last


def _pages(files, pages_str, skip_unreadable):
    """The selected pages of every file, in order; `last` marks a file's last selected page."""
    wanted = set(parse_pages(pages_str)) if pages_str is not None else None
    for f in files:
        try:
            imgs = load_image(f)
        except Exception as e:
            if not skip_unreadable:
                raise
            logger.warning("Skipping %s: %s" % (f, e))
            continue
        keep = [i for i in range(len(imgs)) if wanted is None or i + 1 in wanted]
        if not keep:
            logger.warning("%s: none of its %d page(s) is among --pages %s" % (f, len(imgs), pages_str))
        for k, i in enumerate(keep):
            yield _Page(f, i, imgs[i], k == len(keep) - 1)


def _convert_page(args, fmt, result, img, out_path):
    """One page converted for merge_all_pages (its figures are written with the page's own out_path)."""
    fig = dict(img=img, export_figure=args.figure, figure_dir=args.figure_dir)
    if fmt == "json":
        return export.convert_json(result, out_path, args.ignore_line_break, img, args.figure,
                                   args.figure_dir).model_dump()
    if fmt == "csv":
        return export.convert_csv(result, out_path, args.ignore_line_break, export_figure_letter=args.figure_letter,
                                  **fig)
    convert = export.convert_html if fmt == "html" else export.convert_markdown
    return convert(result, out_path, ignore_line_break=args.ignore_line_break, export_figure_letter=args.figure_letter,
                   figure_width=args.figure_width, **fig)[0]


def _export_page(args, fmt, result, img, out_path):
    """Writes one page's file and its figures."""
    fig = dict(img=img, export_figure=args.figure, figure_dir=args.figure_dir, encoding=args.encoding)
    if fmt == "json":
        export.export_json(result, out_path, ignore_line_break=args.ignore_line_break, **fig)
    elif fmt == "csv":
        export.export_csv(result, out_path, ignore_line_break=args.ignore_line_break,
                          export_figure_letter=args.figure_letter, **fig)
    else:
        write = export.export_html if fmt == "html" else export.export_markdown
        write(result, out_path, ignore_line_break=args.ignore_line_break, export_figure_letter=args.figure_letter,
              figure_width=args.figure_width, **fig)


def _check_input(path):
    path = Path(path)
    if not path.exists():
        raise FileNotFoundError(f"File not found: {path}")
    if path.is_file() and path.suffix[1:].lower() == "pdf":
        load_image(path)            # raises: PDF input is not supported
    return path


def page_batches(path, pages_str, batch_size):
    """The selected pages (--pages) of every file under `path`, in lists of up to `batch_size`.  The next list is
    decoded in a worker thread while the caller works on the current one.  Under a directory, a file that cannot be
    read as a page image is logged and skipped."""
    pages = _pages(input_files(path), pages_str, skip_unreadable=path.is_dir())

    def next_batch():
        batch = []
        for page in pages:
            batch.append(page)
            if len(batch) == batch_size:
                break
        return batch

    with ThreadPoolExecutor(max_workers=1) as decoder:
        pending = decoder.submit(next_batch)
        while True:
            batch = pending.result()
            if not batch:
                return
            pending = decoder.submit(next_batch)
            yield batch


def run(args, analyzer):
    """Analyses every page under `args.arg1` with `analyzer.analyze_pages`, `args.batch` pages per call, and writes
    the outputs.  The next batch is decoded in a worker thread while the analyzer runs on the current one.  Returns the
    paths written (figures not included)."""
    fmt = output_format(args)
    path = _check_input(args.arg1)
    os.makedirs(args.outdir, exist_ok=True)
    logger.info(f"Output directory: {args.outdir}")

    written, combined = [], {}
    start, n_pages = time.time(), 0
    for batch in page_batches(path, args.pages, args.batch):
        results = analyzer.analyze_pages([p.img for p in batch])
        for page, result in zip(batch, results):
            stem = "%s_%s" % (_sanitize_path_component(page.file.parent.name), page.file.stem)
            out_path = os.path.join(args.outdir, "%s_p%d.%s" % (stem, page.index + 1, fmt))
            if not args.combine:
                _export_page(args, fmt, result, page.img, out_path)
                written.append(out_path)
                logger.info(f"Output file: {out_path}")
                continue
            combined.setdefault(page.file, []).append(_convert_page(args, fmt, result, page.img, out_path))
            if page.last:
                out_path = os.path.join(args.outdir, "%s.%s" % (stem, fmt))
                save_merged(fmt, merge_all_pages(fmt, combined.pop(page.file)), out_path, args.encoding)
                written.append(out_path)
                logger.info(f"Output file: {out_path}")
        n_pages += len(batch)
    logger.info("%d page(s) in %.2f sec" % (n_pages, time.time() - start))
    return written


def analyzer_configs(args):
    """DocumentAnalyzer configs from the model options, as yomitoku's command builds them."""
    rec = {"path_cfg": args.tr_cfg}
    configs = {
        "ocr": {"text_detector": {"path_cfg": args.td_cfg}, "text_recognizer": rec},
        "layout_analyzer": {"layout_parser": {"path_cfg": args.lp_cfg},
                            "table_structure_recognizer": {"path_cfg": args.tsr_cfg}},
    }
    if args.lite:
        rec.update(model_name="parseq-tiny-dynw-v4", dynamic_width=True, batch_bucketing=True, source_downscale=True)
    else:
        rec["model_name"] = args.tr_name
        configs["ocr"]["text_detector"]["model_name"] = args.td_name
    if args.enable_rec_orientation_fallback:
        rec.update(rec_orientation_fallback=True, rec_orientation_fallback_thresh=args.rec_orientation_fallback_thresh)
    return configs


def main(argv=None):
    args = build_parser().parse_args(argv)
    output_format(args)
    _check_input(args.arg1)
    from .document_analyzer import DocumentAnalyzer
    analyzer = DocumentAnalyzer(configs=analyzer_configs(args), device=args.device, ignore_meta=args.ignore_meta,
                                reading_order=args.reading_order, ignore_ruby=args.ignore_ruby,
                                ruby_threshold=args.ruby_threshold)
    return run(args, analyzer)
