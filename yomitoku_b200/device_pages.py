"""Pages that are already on the GPU: uint8 CUDA tensors (a `torchvision.io.decode_jpeg(..., device="cuda")` decode,
video frames, an earlier model's output) into the one format every page op reads - BGR pages back to back in a flat
buffer described by a page table (data.page_table) - with one kernel launch (C ABI ytk_pack_pages_u8,
csrc/page_ops.cu) and no host copy.

    dp = device_pages([decode_jpeg(data, device="cuda").permute(1, 2, 0) for data in jpegs], channel_order="rgb")
    results = BatchedOCR(detector, recognizer)(dp)

Every page entry point (TextDetector, TextRecognizer, OCR, BatchedOCR, LayoutParser, TableStructureRecognizer,
CellDetector, LayoutAnalyzer, DocumentAnalyzer) also takes a CUDA (H, W, 3) BGR tensor, or a list of them, and wraps it
with `device_pages`.  After the pack the bytes are those a host page would have been uploaded as, and every later op is
the host path's own, so a page on the device gives exactly the result of the same pixels as a numpy array.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .data import page_table

# Layout of ytk_page_src (include/yomitoku_b200.h): one source page of the pack.
PAGE_SRC_DTYPE = np.dtype([("data", "<u8"), ("sh", "<i8"), ("sw", "<i8"), ("sc", "<i8"), ("H", "<i4"), ("W", "<i4"),
                           ("rgb", "<i4"), ("pad_", "<i4")])

CHANNEL_ORDERS = ("bgr", "rgb")


class DevicePages:
    """Pages in HBM in the page-table layout:
      buf     flat contiguous uint8 CUDA tensor, page i = shapes[i] + (3,) BGR bytes at table[i]["page_off"]
      table   data.PAGE_DTYPE records, one whole page each (= data.page_table(shapes))
      shapes  (h, w) per page
      device  the CUDA device of buf
    `event` is recorded on the stream that wrote buf; `ready(stream)` orders another stream after it."""

    def __init__(self, buf, table, shapes, event=None):
        self.buf, self.table, self.event = buf, table, event
        self.shapes = [(int(h), int(w)) for h, w in shapes]

    @property
    def device(self):
        return self.buf.device

    def __len__(self):
        return len(self.shapes)

    def ready(self, stream=None):
        """Orders `stream` (None: the device's default stream, which the calls without a stream use) after the pack
        and tells the caching allocator that `stream` reads the buffer.  Returns self."""
        s = stream if stream is not None else torch.cuda.default_stream(self.device)
        if self.event is not None:
            s.wait_event(self.event)
        self.buf.record_stream(s)
        return self

    def pair(self):
        """(flat buffer, page table): the form models.as_page_table takes."""
        return self.buf, self.table

    def page(self, i):
        """Page i as an (h, w, 3) view of the buffer."""
        h, w = self.shapes[i]
        o = int(self.table["page_off"][i])
        return self.buf[o:o + h * w * 3].view(h, w, 3)

    def select(self, i):
        """Page i alone as a DevicePages that shares the buffer."""
        h, w = self.shapes[i]
        o = int(self.table["page_off"][i])
        return DevicePages(self.buf[o:o + h * w * 3], page_table([(h, w)])[0], [(h, w)], self.event)

    def numpy(self, i=0):
        """Host copy of page i: the numpy page the same pixels would have been (drawing, host-only fallbacks)."""
        self.ready(torch.cuda.current_stream(self.device))
        return self.page(i).cpu().numpy()


def page_sources(images, channel_order="bgr", need_cuda=True):
    """The checks and the ytk_page_src records of `device_pages`, without a device call: (PAGE_SRC_DTYPE records,
    (h, w) per page, device, page tensors).  Raises ValueError naming the page and the reason."""
    if channel_order not in CHANNEL_ORDERS:
        raise ValueError("channel_order must be 'bgr' or 'rgb', got %r" % (channel_order,))
    if isinstance(images, torch.Tensor):
        if images.dim() != 4:
            raise ValueError("a tensor of pages must be (n, H, W, 3), got shape %s" % (tuple(images.shape),))
        pages = list(images.unbind(0))
    elif isinstance(images, (list, tuple)):
        pages = list(images)
    else:
        raise ValueError("pages must be a list of (H, W, 3) uint8 CUDA tensors or one (n, H, W, 3) tensor, got %s"
                         % type(images).__name__)
    if not pages:
        raise ValueError("no pages")
    recs = np.zeros(len(pages), PAGE_SRC_DTYPE)
    shapes, device = [], None
    for i, p in enumerate(pages):
        if not isinstance(p, torch.Tensor):
            raise ValueError("page %d is a %s, not a torch tensor" % (i, type(p).__name__))
        if need_cuda and not p.is_cuda:
            raise ValueError("page %d is on %s: device pages are CUDA tensors (host pages go in as numpy arrays)"
                             % (i, p.device))
        if device is None:
            device = p.device
        elif p.device != device:
            raise ValueError("page %d is on %s, page 0 on %s: all pages must be on one device" % (i, p.device, device))
        if p.dtype != torch.uint8:
            raise ValueError("page %d has dtype %s: pages are uint8" % (i, p.dtype))
        if p.dim() != 3 or p.shape[2] != 3:
            raise ValueError("page %d has shape %s: pages are (H, W, 3), three channels" % (i, tuple(p.shape)))
        H, W = int(p.shape[0]), int(p.shape[1])
        if H < 1 or W < 1:
            raise ValueError("page %d is empty (%dx%d)" % (i, H, W))
        sh, sw, sc = p.stride()
        recs[i] = (p.data_ptr(), sh, sw, sc, H, W, int(channel_order == "rgb"), 0)
        shapes.append((H, W))
    return recs, shapes, device, pages


def device_pages(images, channel_order="bgr"):
    """images: a list of uint8 CUDA tensors shaped (H, W, 3), of any sizes and strides (a crop, a step or the
    permute(1, 2, 0) of a CHW decode included), or one (n, H, W, 3) tensor; all on one device.  channel_order: "bgr"
    (the convention of the numpy pages of this API) or "rgb" (what torchvision decodes to).  Returns a DevicePages.

    The pack is one launch on the current stream of the pages' device, so it follows whatever wrote them there; the
    engines order their own streams after it (DevicePages.ready).  Anything else raises ValueError with the reason."""
    recs, shapes, device, pages = page_sources(images, channel_order)
    table, total = page_table(shapes)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        buf = torch.empty(total, dtype=torch.uint8, device=device)
        scratch = torch.empty(recs.nbytes + table.nbytes, dtype=torch.uint8, device=device)
        _lib.check(_lib.lib().ytk_pack_pages_u8(recs.ctypes.data, len(recs), buf.data_ptr(), total, table.ctypes.data,
                                                scratch.data_ptr(), scratch.numel(),
                                                ctypes.c_void_p(stream.cuda_stream)))
        for p in pages:
            # a source freed by the caller right away is not reused before the pack has read it, whichever stream
            # allocated it
            p.record_stream(stream)
        event = torch.cuda.Event()
        event.record(stream)
    return DevicePages(buf, table, shapes, event)


def as_device_pages(pages):
    """What a page entry point was given -> DevicePages, or None for host (numpy) input, whose path is unchanged.  A
    DevicePages passes through; a CUDA tensor - one (H, W, 3) page or an (n, H, W, 3) stack - or a list holding CUDA
    tensors is packed as BGR."""
    if isinstance(pages, DevicePages):
        return pages
    if isinstance(pages, torch.Tensor) and pages.is_cuda:
        return device_pages(pages[None] if pages.dim() == 3 else pages)
    if isinstance(pages, (list, tuple)) and any(isinstance(p, torch.Tensor) and p.is_cuda for p in pages):
        return device_pages(pages)
    return None


def require_device(dp, device, who):
    """ValueError unless the pages are on `device` (the model's)."""
    if dp.device != torch.device(device):
        raise ValueError("%s: the pages are on %s, the model runs on %s" % (who, dp.device, torch.device(device)))


def single_page(dp, who):
    if len(dp) != 1:
        raise ValueError("%s takes one page, got %d" % (who, len(dp)))
    return dp


def host_page(img, i=0):
    """Page i as a numpy page: downloaded from DevicePages, else `img` itself."""
    return img.numpy(i) if isinstance(img, DevicePages) else img
