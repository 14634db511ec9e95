"""Searchable PDF out of analysis results: each page image with an invisible, selectable and searchable text layer on top
(reference src/yomitoku/utils/searchable_pdf.py, `create_searchable_pdf`).

    results = analyzer.analyze_pages(dp)                       # dp: a DevicePages, or the numpy / CUDA pages
    create_searchable_pdf(dp, results, "out.pdf", image_quality="middle")

The page images never leave the device as pixels: the pages are resized there (ytk_resize_pages_u8, Pillow's LANCZOS
bit for bit, csrc/resample_ops.cu) and JPEG-encoded by nvJPEG (`torchvision.io.encode_jpeg`, one batched call per
chunk of pages); only the JPEG bytes come back.  A DevicePages that was also given to `DocumentAnalyzer.analyze_pages`
is read in place.  Pages go through in chunks of CHUNK, so a long document holds one chunk of images and of JPEG bytes.

The PDF itself is written here with the standard library only, incrementally and deterministically (no dates, no IDs):
PDF 1.7, a classic xref table, one /DCTDecode image per page drawn over the whole page, and the words as invisible text
(3 Tr) in one Type0 / Identity-H font with no embedded font program - nothing is ever painted - and a /ToUnicode CMap,
so that selecting, copying and searching give the recognised text.  Each word is one text object whose text matrix maps
its run of 1-em codes onto the word's rectangle.

Which words, in which order, follows the reference exactly (`text_layer_words`); what this module does differently is
listed in INTEGRATION.md ("Searchable PDF").
"""
import ctypes
import zlib

import numpy as np
import torch

from . import _lib
from .data import page_table
from .device_pages import DevicePages, device_pages
from .document_analyzer import is_contained

# The reference's presets: (longest side after the resize or None, JPEG quality).
PRESETS = {"high": (None, 85), "middle": (2000, 80), "low": (1500, 60)}
CHUNK = 16

# Layout of ytk_resize_page (include/yomitoku_b200.h).
RESIZE_PAGE_DTYPE = np.dtype([("page_off", "<i8"), ("H", "<i4"), ("W", "<i4"), ("out_w", "<i4"), ("out_h", "<i4"),
                              ("out_off", "<i8")])
LANCZOS, BILINEAR = 1, 2  # YTK_RESAMPLE_*: Pillow's numbering

FONT = "/F1"


def target_size(w, h, image_quality):
    """(width, height) of the page image of a w x h page under a preset, by the reference's own expression."""
    if image_quality not in PRESETS:
        raise ValueError("image_quality must be one of %s, got %r" % (", ".join(PRESETS), image_quality))
    max_long_side = PRESETS[image_quality][0]
    if max_long_side is not None and max(w, h) > max_long_side:
        scale = max_long_side / max(w, h)
        w, h = int(w * scale), int(h * scale)
    if w < 1 or h < 1:
        raise ValueError("a %s page image would be %dx%d pixels: pages this narrow cannot be resized"
                         % (image_quality, w, h))
    return w, h


# ---------------------------------------------------------------------------------------------------------- pages


def _page_list(images):
    """What the page entry points take -> a DevicePages, or a list of numpy / CUDA (H, W, 3) uint8 BGR pages."""
    if isinstance(images, DevicePages):
        return images
    if isinstance(images, np.ndarray):
        images = [images] if images.ndim == 3 else list(images)
    elif isinstance(images, torch.Tensor):
        images = [images] if images.dim() == 3 else list(images.unbind(0))
    elif isinstance(images, (list, tuple)):
        images = list(images)
    else:
        raise ValueError("images must be numpy / CUDA (H, W, 3) uint8 BGR pages, a list of them or a DevicePages, "
                         "got %s" % type(images).__name__)
    for i, p in enumerate(images):
        if isinstance(p, np.ndarray):
            if p.dtype != np.uint8 or p.ndim != 3 or p.shape[2] != 3 or p.shape[0] < 1 or p.shape[1] < 1:
                raise ValueError("page %d: numpy pages are non-empty (H, W, 3) uint8 BGR arrays, got %s %s"
                                 % (i, p.dtype, p.shape))
        elif not (isinstance(p, torch.Tensor) and p.is_cuda):
            raise ValueError("page %d is a %s: pages are numpy arrays or CUDA tensors" % (i, type(p).__name__))
    return images


def _shapes(pages):
    if isinstance(pages, DevicePages):
        return list(pages.shapes)
    return [(int(p.shape[0]), int(p.shape[1])) for p in pages]


def _chunk_on_device(pages, i0, i1):
    """Pages [i0, i1) in HBM: (flat uint8 CUDA buffer, page offsets, shapes).  A DevicePages is read in place."""
    if isinstance(pages, DevicePages):
        pages.ready(torch.cuda.current_stream(pages.device))
        return pages.buf, [int(o) for o in pages.table["page_off"][i0:i1]], pages.shapes[i0:i1]
    part = pages[i0:i1]
    if all(isinstance(p, torch.Tensor) for p in part):
        dp = device_pages(part)
        dp.ready(torch.cuda.current_stream(dp.device))
        return dp.buf, [int(o) for o in dp.table["page_off"]], dp.shapes
    if any(isinstance(p, torch.Tensor) for p in part):
        raise ValueError("pages %d..%d mix numpy arrays and CUDA tensors" % (i0, i1 - 1))
    shapes = _shapes(part)
    table, total = page_table(shapes)
    host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for p, off in zip(part, table["page_off"]):
        hv[int(off):int(off) + p.size] = np.ascontiguousarray(p).reshape(-1)
    buf = host.to("cuda", non_blocking=True)
    return buf, [int(o) for o in table["page_off"]], shapes


def resize_pages(buf, page_offs, shapes, sizes):
    """The pages of `buf` (flat uint8 CUDA buffer, BGR page i of shapes[i] = (H, W) at page_offs[i]) resized to
    sizes[i] = (w, h) on the device, one launch pair on the current stream: a list of planar (3, h, w) uint8 RGB views
    of one output buffer, Image.fromarray(rgb).resize((w, h), Image.LANCZOS) bit for bit."""
    recs = np.zeros(len(shapes), RESIZE_PAGE_DTYPE)
    off = 0
    for i, ((H, W), (w, h)) in enumerate(zip(shapes, sizes)):
        recs[i] = (page_offs[i], H, W, w, h, off)
        off += 3 * w * h
    L = _lib.lib()
    need = L.ytk_resize_pages_scratch_bytes(recs.ctypes.data, len(recs), LANCZOS)
    if need < 0:
        raise ValueError(L.ytk_last_error().decode())
    out = torch.empty(off, dtype=torch.uint8, device=buf.device)
    scratch = torch.empty(max(need, 1), dtype=torch.uint8, device=buf.device)
    stream = torch.cuda.current_stream(buf.device)
    _lib.check(L.ytk_resize_pages_u8(buf.data_ptr(), buf.numel(), recs.ctypes.data, len(recs), LANCZOS,
                                     scratch.data_ptr(), scratch.numel(), out.data_ptr(), out.numel(),
                                     ctypes.c_void_p(stream.cuda_stream)))
    return [out[int(r["out_off"]):int(r["out_off"]) + 3 * int(r["out_w"]) * int(r["out_h"])]
            .view(3, int(r["out_h"]), int(r["out_w"])) for r in recs]


def encode_pages(images, image_quality="high", chunk=CHUNK):
    """Yields (JPEG bytes, (w, h) of the JPEG, (W, H) of the page) per page, in order, `chunk` pages at a time: one
    resize launch pair and one batched nvJPEG encode per chunk."""
    from torchvision.io import encode_jpeg  # only this module needs torchvision

    pages = _page_list(images)
    shapes = _shapes(pages)
    sizes = [target_size(W, H, image_quality) for H, W in shapes]
    q = PRESETS[image_quality][1]
    for i0 in range(0, len(shapes), chunk):
        i1 = min(i0 + chunk, len(shapes))
        buf, offs, sh = _chunk_on_device(pages, i0, i1)
        with torch.cuda.device(buf.device):
            planar = resize_pages(buf, offs, sh, sizes[i0:i1])
            jpegs = encode_jpeg(planar, quality=q)
            data = [j.cpu().numpy().tobytes() for j in jpegs]
        for k, d in enumerate(data):
            H, W = sh[k]
            yield d, sizes[i0 + k], (W, H)


# ------------------------------------------------------------------------------------------------ the text layer


def _poly2rect(points):
    """[x_min, y_min, x_max, y_max] of a quad, int-truncated as the reference does."""
    p = np.array(points, dtype=int)
    return [int(p[:, 0].min()), int(p[:, 1].min()), int(p[:, 0].max()), int(p[:, 1].max())]


def text_layer_words(doc):
    """The words of one page's result in the reference's text-layer order: the containers (paragraphs, sub-order 0;
    table cells, sub-order (row, col); figure paragraphs, sub-order = index) sorted by (order, sub-order), and in each
    the words whose rectangle it holds (is_contained(container box, rect, 0.7)), sorted by (-x_min, y_min) in a vertical
    container and by (y_min, x_min) otherwise.  A word in two containers comes twice, a word in none not at all."""
    containers = []
    for p in doc.paragraphs:
        containers.append((p.box, p.order, 0, p.direction))
    for t in doc.tables:
        for cell in t.cells:
            containers.append((cell.box, t.order, (cell.row, cell.col), "horizontal"))
    for f in doc.figures:
        for k, p in enumerate(f.paragraphs):
            containers.append((p.box, f.order, k, p.direction))
    containers = sorted(containers, key=lambda c: (c[1], c[2]))
    rects = [_poly2rect(w.points) for w in doc.words]
    out = []
    for box, _, _, direction in containers:
        inside = [k for k, r in enumerate(rects) if is_contained(box, r, 0.7)]
        if direction == "vertical":
            inside.sort(key=lambda k: (-rects[k][0], rects[k][1]))
        else:
            inside.sort(key=lambda k: (rects[k][1], rects[k][0]))
        out.extend(doc.words[k] for k in inside)
    return out


def _num(v):
    """A PDF number: an integer as such, anything else with 9 decimals, trailing zeros dropped."""
    if float(v) == int(v):
        return "%d" % int(v)
    return ("%.9f" % v).rstrip("0").rstrip(".")


def word_matrix(rect, n, page_h, vertical):
    """Text matrix mapping a run of n 1-em codes (font size 1) onto rect = (x1, y1, x2, y2) in page pixels (y down)
    on a page of height page_h (PDF y up).  Vertical runs go top to bottom with the glyphs' up pointing right."""
    x1, y1, x2, y2 = rect
    if vertical:
        return (0, -(y2 - y1) / n, x2 - x1, 0, x1, page_h - y1)
    return ((x2 - x1) / n, 0, 0, y2 - y1, x1, page_h - y2)


class _Codes:
    """The document's character table: code i (2 bytes, /Identity-H) -> character; codes start at 1."""

    def __init__(self):
        self.code = {}

    def encode(self, text):
        out = []
        for ch in text:
            c = self.code.get(ch)
            if c is None:
                c = len(self.code) + 1
                if c > 0xFFFF:
                    raise ValueError("more than 65535 distinct characters in one document")
                self.code[ch] = c
            out.append(c)
        return out

    def to_unicode(self):
        lines = ["/CIDInit /ProcSet findresource begin", "12 dict begin", "begincmap",
                 "/CIDSystemInfo << /Registry (Adobe) /Ordering (UCS) /Supplement 0 >> def",
                 "/CMapName /Adobe-Identity-UCS def", "/CMapType 2 def",
                 "1 begincodespacerange", "<0000> <FFFF>", "endcodespacerange"]
        items = sorted((c, ch) for ch, c in self.code.items())
        for k in range(0, len(items), 100):
            block = items[k:k + 100]
            lines.append("%d beginbfchar" % len(block))
            lines.extend("<%04X> <%s>" % (c, ch.encode("utf-16-be").hex().upper()) for c, ch in block)
            lines.append("endbfchar")
        lines += ["endcmap", "CMapName currentdict /CMap defineresource pop", "end", "end"]
        return ("\n".join(lines) + "\n").encode("ascii")


def page_content(words, page_w, page_h, codes, image="/Im0"):
    """The content stream of one page: the image over the whole page, then one invisible text object per word."""
    ops = ["q %s 0 0 %s 0 0 cm %s Do Q" % (_num(page_w), _num(page_h), image)]
    for w in words:
        text = w.content
        rect = _poly2rect(w.points)
        if not text or rect[2] <= rect[0] or rect[3] <= rect[1]:
            continue
        cs = codes.encode(text)
        m = word_matrix(rect, len(cs), page_h, w.direction == "vertical")
        ops.append("BT 3 Tr %s 1 Tf %s Tm <%s> Tj ET" % (FONT, " ".join(_num(v) for v in m),
                                                         "".join("%04X" % c for c in cs)))
    return ("\n".join(ops) + "\n").encode("ascii")


class PdfWriter:
    """Writes a PDF 1.7 file object by object as they arrive (offsets recorded), then the xref table, the trailer and
    startxref.  Object numbers are reserved up front where an object is referred to before it is written."""

    def __init__(self, f):
        self.f = f
        self.pos = 0
        self.offsets = {}
        self.next = 1
        self._put(b"%PDF-1.7\n%\xe2\xe3\xcf\xd3\n")

    def _put(self, b):
        self.f.write(b)
        self.pos += len(b)

    def reserve(self):
        n = self.next
        self.next += 1
        return n

    def obj(self, n, body):
        self.offsets[n] = self.pos
        self._put(b"%d 0 obj\n" % n + body.encode("ascii") + b"\nendobj\n")

    def stream(self, n, entries, data):
        self.offsets[n] = self.pos
        self._put(b"%d 0 obj\n<< %s /Length %d >>\nstream\n" % (n, entries.encode("ascii"), len(data)) + data +
                  b"\nendstream\nendobj\n")

    def close(self, root):
        size = self.next
        missing = [n for n in range(1, size) if n not in self.offsets]
        assert not missing, missing
        xref = self.pos
        rows = [b"xref\n0 %d\n" % size, b"0000000000 65535 f \n"]
        rows += [b"%010d 00000 n \n" % self.offsets[n] for n in range(1, size)]
        self._put(b"".join(rows))
        self._put(b"trailer\n<< /Size %d /Root %d 0 R >>\nstartxref\n%d\n%%%%EOF\n" % (size, root, xref))


def write_pdf(f, pages, docs):
    """Writes the PDF to the binary file f.  pages: iterable of (JPEG bytes, (w, h) of the JPEG, (W, H) of the page);
    docs: one analysis result per page."""
    w = PdfWriter(f)
    catalog, page_tree, font, cid_font, descriptor, to_unicode = (w.reserve() for _ in range(6))
    w.obj(catalog, "<< /Type /Catalog /Pages %d 0 R >>" % page_tree)
    w.obj(font, "<< /Type /Font /Subtype /Type0 /BaseFont /YomitokuText /Encoding /Identity-H /DescendantFonts "
                "[%d 0 R] /ToUnicode %d 0 R >>" % (cid_font, to_unicode))
    w.obj(cid_font, "<< /Type /Font /Subtype /CIDFontType2 /BaseFont /YomitokuText /CIDSystemInfo << /Registry "
                    "(Adobe) /Ordering (Identity) /Supplement 0 >> /FontDescriptor %d 0 R /DW 1000 /CIDToGIDMap "
                    "/Identity >>" % descriptor)
    w.obj(descriptor, "<< /Type /FontDescriptor /FontName /YomitokuText /Flags 4 /FontBBox [0 0 1000 1000] "
                      "/ItalicAngle 0 /Ascent 1000 /Descent 0 /CapHeight 1000 /StemV 80 >>")
    codes = _Codes()
    kids = []
    for (jpeg, (iw, ih), (W, H)), doc in zip(pages, docs):
        image, content, page = w.reserve(), w.reserve(), w.reserve()
        w.stream(image, "/Type /XObject /Subtype /Image /Width %d /Height %d /ColorSpace /DeviceRGB "
                        "/BitsPerComponent 8 /Filter /DCTDecode" % (iw, ih), jpeg)
        w.stream(content, "/Filter /FlateDecode", zlib.compress(page_content(text_layer_words(doc), W, H, codes), 6))
        w.obj(page, "<< /Type /Page /Parent %d 0 R /MediaBox [0 0 %d %d] /Resources << /Font << %s %d 0 R >> "
                    "/XObject << /Im0 %d 0 R >> >> /Contents %d 0 R >>" % (page_tree, W, H, FONT, font, image,
                                                                           content))
        kids.append(page)
    w.obj(page_tree, "<< /Type /Pages /Kids [%s] /Count %d >>" % (" ".join("%d 0 R" % k for k in kids), len(kids)))
    w.stream(to_unicode, "", codes.to_unicode())
    w.close(catalog)


def create_searchable_pdf(images, docs, output_path, font_path=None, image_quality="high"):
    """The reference's create_searchable_pdf: writes the pages `images` (numpy or CUDA (H, W, 3) uint8 BGR pages, a
    list of them, or a DevicePages) with the text layer of `docs` (one DocumentAnalyzerSchema per page) to
    output_path.  image_quality: "high" (the page as it is, JPEG quality 85), "middle" (longest side at most 2000, 80)
    or "low" (1500, 60).  font_path must be None: no font is embedded (the text is never painted).  Raises ValueError
    for an unknown preset, a page count other than len(docs), or a page image below 1 pixel."""
    if font_path is not None:
        raise ValueError("font_path must be None: the text layer is invisible and embeds no font")
    if image_quality not in PRESETS:
        raise ValueError("image_quality must be one of %s, got %r" % (", ".join(PRESETS), image_quality))
    pages = _page_list(images)
    docs = list(docs)
    if len(pages) != len(docs):
        raise ValueError("%d pages but %d results" % (len(pages), len(docs)))
    if not docs:
        raise ValueError("no pages")
    for H, W in _shapes(pages):
        target_size(W, H, image_quality)
    with open(output_path, "wb") as f:
        write_pdf(f, encode_pages(pages, image_quality), docs)
