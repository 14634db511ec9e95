"""CPU: the searchable-PDF writer (yomitoku_b200/searchable_pdf.py) read back by the small PDF reader below - header,
xref, trailer, stream lengths, image size against the JPEG's SOF header, the ToUnicode CMap, the text layer's words and
their text matrices - the text-layer order against the reference's own create_searchable_pdf (tests/golden/pdf_ref.json,
tests/golden/make_golden_pdf.py), and the refused inputs.  The device path (resize, nvJPEG) is in
tests/test_gpu_searchable_pdf.py."""
import io
import json
import os
import re
import types
import zlib

import cv2
import numpy as np
import pytest

from yomitoku_b200 import create_searchable_pdf
from yomitoku_b200.searchable_pdf import _poly2rect, text_layer_words, write_pdf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pdf_ref.json")


# ------------------------------------------------------------------------------------------------- a small reader
class Pdf:
    def __init__(self, data):
        self.data = data
        assert data.startswith(b"%PDF-1.7\n%")
        assert all(b >= 128 for b in data[10:14]) and data[14:15] == b"\n"    # the binary comment
        m = re.search(rb"startxref\n(\d+)\n%%EOF\n$", data)
        self.xref = int(m.group(1))
        assert data[self.xref:self.xref + 5] == b"xref\n"
        head = re.match(rb"xref\n0 (\d+)\n", data[self.xref:])
        self.size = int(head.group(1))
        rows = data[self.xref + head.end():]
        self.offsets = {}
        for n in range(self.size):
            row = rows[20 * n:20 * n + 20]
            assert len(row) == 20 and row.endswith(b" \n"), row
            if n == 0:
                assert row == b"0000000000 65535 f \n"
                continue
            assert re.fullmatch(rb"\d{10} 00000 n \n", row), row
            self.offsets[n] = int(row[:10])
        trailer = rows[20 * self.size:]
        t = re.match(rb"trailer\n<< /Size (\d+) /Root (\d+) 0 R >>\nstartxref\n", trailer)
        assert int(t.group(1)) == self.size
        self.root = int(t.group(2))
        self.objs = {n: self._parse(n, o) for n, o in self.offsets.items()}

    def _parse(self, n, off):
        head = b"%d 0 obj\n" % n
        assert self.data[off:off + len(head)] == head, (n, self.data[off:off + 20])
        body = self.data[off + len(head):]
        if body.startswith(b"<<") and re.match(rb"<<[^\n]*>>\nstream\n", body):
            d = re.match(rb"(<<[^\n]*>>)\nstream\n", body)
            length = int(re.search(rb"/Length (\d+) >>$", d.group(1)).group(1))
            s = body[d.end():d.end() + length]
            tail = b"\nendstream\nendobj\n"
            assert body[d.end() + length:d.end() + length + len(tail)] == tail   # /Length is exact
            return d.group(1).decode(), s
        end = body.index(b"\nendobj\n")
        return body[:end].decode(), None

    def ref(self, n, key):
        return int(re.search(r"%s (\d+) 0 R" % key, self.objs[n][0]).group(1))

    def pages(self):
        tree = self.ref(self.root, "/Pages")
        kids = [int(k) for k in re.findall(r"(\d+) 0 R", re.search(r"/Kids \[([^\]]*)\]", self.objs[tree][0]).group(1))]
        assert int(re.search(r"/Count (\d+)", self.objs[tree][0]).group(1)) == len(kids)
        return kids

    def content(self, page):
        d, s = self.objs[self.ref(page, "/Contents")]
        return zlib.decompress(s).decode("ascii") if "/FlateDecode" in d else s.decode("ascii")


def parse_to_unicode(cmap):
    text = cmap.decode("ascii")
    assert "begincmap" in text and "endcmap" in text
    assert "1 begincodespacerange\n<0000> <FFFF>\nendcodespacerange" in text
    table = {}
    for count, block in re.findall(r"(\d+) beginbfchar\n(.*?)endbfchar", text, flags=re.S):
        lines = block.strip().split("\n")
        assert int(count) == len(lines) <= 100
        for line in lines:
            m = re.fullmatch(r"<([0-9A-F]{4})> <((?:[0-9A-F]{4})+)>", line)
            assert m, line
            table[int(m.group(1), 16)] = bytes.fromhex(m.group(2)).decode("utf-16-be")
    return table


WORD = re.compile(r"BT 3 Tr /F1 1 Tf (\S+) (\S+) (\S+) (\S+) (\S+) (\S+) Tm <([0-9A-F]*)> Tj ET")


def text_layer(pdf):
    font = pdf.ref(pdf.pages()[0], "/F1")
    to_unicode = parse_to_unicode(pdf.objs[pdf.ref(font, "/ToUnicode")][1])
    out = []
    for page in pdf.pages():
        words = []
        for m in WORD.finditer(pdf.content(page)):
            codes = [int(m.group(7)[k:k + 4], 16) for k in range(0, len(m.group(7)), 4)]
            assert all(c in to_unicode for c in codes)
            words.append(("".join(to_unicode[c] for c in codes), [float(m.group(k)) for k in range(1, 7)], len(codes)))
        out.append(words)
    return out


def jpeg_size(data):
    k = 2
    while k < len(data):
        assert data[k] == 0xFF
        marker, length = data[k + 1], int.from_bytes(data[k + 2:k + 4], "big")
        if marker in (0xC0, 0xC1, 0xC2):
            return (int.from_bytes(data[k + 7:k + 9], "big"), int.from_bytes(data[k + 5:k + 7], "big"), data[k + 9])
        k += 2 + length
    raise AssertionError("no SOF")


# -------------------------------------------------------------------------------------------------------- cases
def _ns(v):
    if isinstance(v, dict):
        return types.SimpleNamespace(**{k: _ns(x) for k, x in v.items()})
    if isinstance(v, list) and v and isinstance(v[0], dict):
        return [_ns(x) for x in v]
    return v


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN, encoding="utf-8") as f:
        return json.load(f)


def _write(pages, docs):
    buf = io.BytesIO()
    write_pdf(buf, pages, docs)
    return buf.getvalue()


def _jpeg(w, h, seed):
    img = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 80])[1].tobytes()


def _golden_pdf(golden):
    pages, docs = [], []
    for k, p in enumerate(golden["pages"]):
        W, H = p["shape"]["W"], p["shape"]["H"]
        iw, ih = (W, H) if k % 2 == 0 else (W // 2, H // 2)     # resized page images on odd pages
        pages.append((_jpeg(iw, ih, k), (iw, ih), (W, H)))
        docs.append(_ns(p["doc"]))
    return pages, docs


def test_structure(golden):
    pages, docs = _golden_pdf(golden)
    data = _write(pages, docs)
    pdf = Pdf(data)
    assert sorted(pdf.objs) == list(range(1, pdf.size))
    kids = pdf.pages()
    assert len(kids) == len(pages)
    for page, (jpeg, (iw, ih), (W, H)) in zip(kids, pages):
        d = pdf.objs[page][0]
        assert "/MediaBox [0 0 %d %d]" % (W, H) in d
        image = int(re.search(r"/Im0 (\d+) 0 R", d).group(1))
        idict, istream = pdf.objs[image]
        assert istream == jpeg
        assert "/Filter /DCTDecode" in idict and "/ColorSpace /DeviceRGB" in idict and "/BitsPerComponent 8" in idict
        w, h, comps = jpeg_size(istream)
        assert (w, h, comps) == (iw, ih, 3)
        assert "/Width %d /Height %d" % (w, h) in idict
        assert pdf.content(page).startswith("q %d 0 0 %d 0 0 cm /Im0 Do Q\n" % (W, H))   # image over the whole page
    font = pdf.ref(kids[0], "/F1")
    assert "/Subtype /Type0" in pdf.objs[font][0] and "/Encoding /Identity-H" in pdf.objs[font][0]
    cid = int(re.search(r"/DescendantFonts \[(\d+) 0 R\]", pdf.objs[font][0]).group(1))
    for key in ("/Subtype /CIDFontType2", "/DW 1000", "/CIDToGIDMap /Identity"):
        assert key in pdf.objs[cid][0]
    desc = pdf.ref(cid, "/FontDescriptor")
    assert "/FontFile" not in pdf.objs[desc][0]                                  # no font program
    assert _write(*_golden_pdf(golden)) == data                                  # deterministic


def _expected(doc):
    return [w for w in text_layer_words(doc) if w.content and _area(_poly2rect(w.points)) > 0]


def _area(r):
    return max(0, r[2] - r[0]) * max(0, r[3] - r[1])


def test_text_layer_words_and_matrices(golden):
    pages, docs = _golden_pdf(golden)
    layer = text_layer(Pdf(_write(pages, docs)))
    seen_vertical = seen_non_bmp = False
    for (_, _, (W, H)), doc, words in zip(pages, docs, layer):
        want = _expected(doc)
        assert [t for t, _, _ in words] == [w.content for w in want]
        for (text, m, n), w in zip(words, want):
            x1, y1, x2, y2 = _poly2rect(w.points)
            a, b, c, d, e, f = m
            # the run's corners (0, 0), (n, 0), (0, 1) in text space
            p0, pn, p1 = (e, f), (a * n + e, b * n + f), (c + e, d + f)
            if w.direction == "vertical":
                seen_vertical = True
                want_pts = ((x1, H - y1), (x1, H - y2), (x2, H - y1))
            else:
                want_pts = ((x1, H - y2), (x2, H - y2), (x1, H - y1))
            for got, exp in zip((p0, pn, p1), want_pts):
                assert abs(got[0] - exp[0]) <= 1e-6 and abs(got[1] - exp[1]) <= 1e-6, (text, got, exp)
            seen_non_bmp |= any(ord(ch) > 0xFFFF for ch in text)
    assert seen_vertical and seen_non_bmp


def test_order_equals_reference(golden):
    """The words the reference considers, in its order, are text_layer_words; what it draws - a vertical word's
    per-character draws joined - is the text layer, except the documented skips (empty text, zero-area rectangle)."""
    pages, docs = _golden_pdf(golden)
    layer = text_layer(Pdf(_write(pages, docs)))
    total = 0
    for p, doc, words in zip(golden["pages"], docs, layer):
        considered = text_layer_words(doc)
        assert [w.content for w in considered] == [c["text"] for c in p["considered"]]
        drawn = [d["text"] for d in p["drawn"]]
        keep = [c["text"] for c in p["considered"] if c["extents"][0] > 0 and c["extents"][1] > 0]
        assert drawn == keep                          # the reference skips a word whose font size comes out 0
        kept = [w for c, w in zip(p["considered"], considered) if c["extents"][0] > 0 and c["extents"][1] > 0]
        assert [d["vertical"] for d in p["drawn"] if d["text"]] == [w.direction == "vertical" for w in kept if w.content]
        assert [t for t, _, _ in words] == [t for t in drawn if t]   # ... and this module an empty word too
        total += len(words)
    assert total >= 30


def test_to_unicode_blocks_of_100():
    chars = [chr(0x4E00 + k) for k in range(230)] + ["😀", "𠮷"]
    doc = _ns({"paragraphs": [{"box": [0, 0, 1000, 1000], "order": 0, "direction": "horizontal"}], "tables": [],
               "figures": [], "words": [{"points": [[10, 10 + 3 * k], [20, 10 + 3 * k], [20, 12 + 3 * k],
                                                    [10, 12 + 3 * k]], "content": ch, "direction": "horizontal"}
                                        for k, ch in enumerate(chars)]})
    pdf = Pdf(_write([(_jpeg(8, 8, 0), (8, 8), (1000, 1000))], [doc]))
    font = pdf.ref(pdf.pages()[0], "/F1")
    cmap = pdf.objs[pdf.ref(font, "/ToUnicode")][1]
    assert re.findall(rb"(\d+) beginbfchar", cmap) == [b"100", b"100", b"32"]
    assert sorted(parse_to_unicode(cmap).values()) == sorted(chars)
    assert [t for t, _, _ in text_layer(pdf)[0]] == chars


def test_refused_inputs(tmp_path):
    page = np.zeros((20, 30, 3), np.uint8)
    doc = _ns({"paragraphs": [], "tables": [], "figures": [], "words": []})
    out = str(tmp_path / "x.pdf")
    with pytest.raises(ValueError, match="font_path"):
        create_searchable_pdf([page], [doc], out, font_path="font.ttf")
    with pytest.raises(ValueError, match="image_quality"):
        create_searchable_pdf([page], [doc], out, image_quality="best")
    with pytest.raises(ValueError, match="2 pages but 1 results"):
        create_searchable_pdf([page, page], [doc], out)
    with pytest.raises(ValueError, match="1 pages but 2 results"):
        create_searchable_pdf(page, [doc, doc], out)
    with pytest.raises(ValueError, match="pixels"):
        create_searchable_pdf([np.zeros((1, 2100, 3), np.uint8)], [doc], out, image_quality="middle")
    with pytest.raises(ValueError, match="uint8"):
        create_searchable_pdf([page.astype(np.float32)], [doc], out)
    with pytest.raises(ValueError, match="images must be"):
        create_searchable_pdf("page.png", [doc], out)
    with pytest.raises(ValueError, match="no pages"):
        create_searchable_pdf([], [], out)
    assert not os.path.exists(out)
