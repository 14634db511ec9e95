"""LayoutAnalyzer = LayoutParser + TableStructureRecognizer (reference src/yomitoku/layout_analyzer.py:7-49): the
`layout_analyzer` DocumentAnalyzer builds by default when a GPU is present."""
import torch

from .device_pages import as_device_pages
from .layout_parser import LayoutParser, upload_pages
from .schemas import LayoutAnalyzerSchema
from .table_structure_recognizer import TableStructureRecognizer


class LayoutAnalyzer:
    def __init__(self, configs={}, device="cuda", visualize=False):
        if not isinstance(configs, dict):
            raise ValueError("configs must be a dict. See the https://kotaro-kinoshita.github.io/yomitoku-dev/usage/")
        parser_kw = {"device": device, "visualize": visualize, **configs.get("layout_parser", {})}
        table_kw = {"device": device, "visualize": visualize, **configs.get("table_structure_recognizer", {})}
        self.layout_parser = LayoutParser(**parser_kw)
        self.table_structure_recognizer = TableStructureRecognizer(**table_kw)

    def __call__(self, img):
        """img: BGR page (numpy, or on the GPU: a CUDA (H, W, 3) uint8 tensor or a one-page DevicePages)."""
        dp = as_device_pages(img)
        if dp is not None:
            # a page already in HBM: the parser and the table batch both read the packed buffer
            layout, vis = self.layout_parser(dp)
            tables, vis = self.table_structure_recognizer(dp, [t.box for t in layout.tables], vis=vis)
            return LayoutAnalyzerSchema(paragraphs=layout.paragraphs, tables=tables, figures=layout.figures), vis
        # on a CUDA device the page goes up once as u8: the parser and the table batch both read that buffer
        page_dev = upload_pages([img], self.layout_parser.model)
        layout, vis = self.layout_parser(img, pages_dev=page_dev)
        tables, vis = self.table_structure_recognizer(img, [t.box for t in layout.tables], vis=vis, pages_dev=page_dev)
        return LayoutAnalyzerSchema(paragraphs=layout.paragraphs, tables=tables, figures=layout.figures), vis

    def analyze_pages(self, pages):
        """Batched entry (new surface): every page's layout in one device call, then one table batch per page.  On a
        CUDA device every page goes up once; each page's table batch reads its slice of that buffer.  Pages already on
        the GPU (CUDA tensors or a DevicePages) are read where they are."""
        dp = as_device_pages(pages)
        if dp is not None:
            out = []
            for i, layout in enumerate(self.layout_parser.parse_pages(dp)):
                tables, _ = self.table_structure_recognizer(dp.select(i), [t.box for t in layout.tables])
                out.append(LayoutAnalyzerSchema(paragraphs=layout.paragraphs, tables=tables, figures=layout.figures))
            return out
        pages_dev = upload_pages(pages, self.layout_parser.model)
        views = [None] * len(pages)
        if pages_dev is not None:
            views = list(torch.split(pages_dev, [p.size for p in pages]))
        out = []
        for page, view, layout in zip(pages, views, self.layout_parser.parse_pages(pages, pages_dev)):
            tables, _ = self.table_structure_recognizer(page, [t.box for t in layout.tables], pages_dev=view)
            out.append(LayoutAnalyzerSchema(paragraphs=layout.paragraphs, tables=tables, figures=layout.figures))
        return out
