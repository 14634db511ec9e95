"""Command line: `python -m yomitoku_b200.extract <file-or-dir> -s schema.yaml -o results`.

Options, defaults and output file names follow yomitoku's `yomitoku_extract` command (src/yomitoku/cli/
extract_rule.py); what differs is how the pages run.  The pages of all input files go through
`TableSemanticParser.extract_pages` in batches of `--batch` pages (of any mix of sizes), while one thread decodes the
next batch (the file walk, --pages and the batching are the document command's, cli.py).  Each page's file is what
`extractor.extract` returns for that page alone:

    <outdir>/<stem>_p<N>_extract.json      N counts from 1; {name: value} with --simple

A file in a directory that cannot be read as a page image is logged and skipped.  A missing input or schema file, or
a schema that does not validate, is an error before any model is built.

Not available here: the extraction picture (-v), which needs a TrueType font this package does not ship, and PDF
input (--dpi), for which there is no PDF renderer among the dependencies.
"""
import argparse
import json
import os
import sys
import time
import types
from pathlib import Path

from . import extractor
from .base import set_logger
from .cli import SUPPORT_ENCODING, _check_input, page_batches
from .extractor import ExtractionSchema

logger = set_logger(__name__, "INFO")


def build_parser():
    p = argparse.ArgumentParser(prog="python -m yomitoku_b200.extract",
                                description="Extract the fields of a YAML schema from form images by rule-based "
                                            "matching over the table semantic parser's results.")
    p.add_argument("input", type=str, help="input image file or directory (searched recursively)")
    p.add_argument("-s", "--schema", type=str, required=True, help="extraction schema file (YAML)")
    p.add_argument("-o", "--outdir", type=str, default="results", help="output directory (default: results)")
    p.add_argument("-d", "--device", type=str, default="cuda", help="device for TableSemanticParser (default: cuda)")
    p.add_argument("-l", "--lite", action="store_true",
                   help="use the lite recognizer (parseq-tiny-dynw-v4 with dynamic-width batching)")
    p.add_argument("-v", "--vis", action="store_true",
                   help="not available: the extraction picture needs a TrueType font this package does not ship")
    p.add_argument("--cell-detector-model", type=str, default="rtdetrv2", choices=["rtdetrv2"],
                   help="cell detector model (rtdetrv2: input size 960)")
    p.add_argument("--no-normalize", action="store_true", help="skip the schema's normalisation rules")
    p.add_argument("--simple", action="store_true", help="write {name: value} without boxes and metadata")
    p.add_argument("--pages", type=str, default=None, help="pages to process, e.g. 1,2,5-10 (default: all)")
    p.add_argument("--encoding", type=str, default="utf-8",
                   help="character encoding of the output files (%s); characters it cannot represent are dropped"
                   % ", ".join(SUPPORT_ENCODING))
    p.add_argument("--batch", type=int, default=16, help="pages per extract_pages call (default: 16)")
    return p


def check_args(args):
    """Refuses what this command cannot do and loads the schema, before any model is built.  Returns (input path,
    ExtractionSchema)."""
    if args.vis:
        raise ValueError("-v/--vis is not available in this package: the extraction picture needs a TrueType font "
                         "it does not ship")
    if args.encoding not in SUPPORT_ENCODING:
        raise ValueError(f"Invalid encoding: {args.encoding}")
    if args.batch < 1:
        raise ValueError(f"--batch must be at least 1, got {args.batch}")
    path = _check_input(args.input)
    if not Path(args.schema).is_file():
        raise FileNotFoundError(f"Schema file not found: {args.schema}")
    schema = ExtractionSchema.from_yaml(args.schema)
    logger.info(f"Loaded schema with {len(schema.fields)} fields")
    return path, schema


def run(args, parser):
    """Extracts the schema's fields from every page under `args.input` with `parser.extract_pages`, `args.batch` pages
    per call, and writes one JSON file per page.  Returns the paths written."""
    path, schema = check_args(args)
    os.makedirs(args.outdir, exist_ok=True)
    written = []
    start, n_pages = time.time(), 0
    for batch in page_batches(path, args.pages, args.batch):
        outputs = parser.extract_pages([p.img for p in batch], schema, normalize=not args.no_normalize,
                                       simple=args.simple)
        for page, out in zip(batch, outputs):
            out_path = os.path.join(args.outdir, "%s_p%d_extract.json" % (page.file.stem, page.index + 1))
            with open(out_path, "w", encoding=args.encoding, errors="ignore") as f:
                json.dump(out, f, ensure_ascii=False, indent=2)
            written.append(out_path)
            logger.info(f"Output JSON: {out_path}")
        n_pages += len(batch)
    logger.info("%d page(s) in %.2f sec" % (n_pages, time.time() - start))
    return written


def parser_configs(args):
    """TableSemanticParser configs from the model options, as yomitoku's command builds them."""
    configs = {"table_cell_parser": {"model_name": args.cell_detector_model}}
    if args.lite:
        configs["text_recognizer"] = {"model_name": "parseq-tiny-dynw-v4", "dynamic_width": True,
                                      "batch_bucketing": True}
    return configs


def main(argv=None):
    args = build_parser().parse_args(argv)
    check_args(args)
    from .table_semantic_parser import TableSemanticParser
    return run(args, TableSemanticParser(configs=parser_configs(args), device=args.device))


class _CommandModule(types.ModuleType):
    """`yomitoku_b200.extract` names both this module and the package's `extract` function (extractor.extract).
    Importing this module rebinds the package attribute to the module, so calling the module calls the function."""

    def __call__(self, *args, **kwargs):
        return extractor.extract(*args, **kwargs)


sys.modules[__name__].__class__ = _CommandModule

if __name__ == "__main__":
    main()
