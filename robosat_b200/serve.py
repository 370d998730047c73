"""Single-image latency path: the H100 replacement for `Predictor.segment` of `rs serve`
(robosat/tools/serve.py:135-192).

Reference: PIL image -> ConvertImageMode("RGB") -> ImageToTensor -> Normalize -> net(batch of 1) -> .cpu().numpy()
-> argmax(axis=0).astype(uint8) -> P-mode image with the dataset's palette.

Here the whole device side of that call -- H2D copy of the raw uint8 pixels from a pinned buffer, normalisation, the U-Net plan
(60 launches), the per-pixel argmax and the D2H copy of one byte per pixel -- is captured ONCE into a CUDA graph and replayed per
request. The kernels already chain through programmatic dependent launch, so the graph buys little GPU time; what it does buy
is one driver call instead of 63 ctypes launches per request and immunity to host jitter. Weights, activations
and both pinned staging buffers are static. `use_graph=False` serves from the stream with identical results (tests/test_serve_gpu.py).
"""

import numpy as np
import torch
from PIL import Image

from robosat_b200 import _lib
from robosat_b200 import tta as tta_mod
from robosat_b200.colors import make_palette
from robosat_b200.engine import UNetEngine


class SegmentEngine:
    """uint8 RGB tiles [B, H, W, 3] (host) -> uint8 class-index masks [B, H, W] (host), graph-replayed."""

    def __init__(self, state_dict, num_classes, height, width, batch=1, device="cuda", use_graph=True, precision=None, tta="none"):
        """tta="flip" | "d4": the mask is the argmax of the mean probability over 2 | 8 dihedral views (robosat_b200/tta.py), all
        of them in one engine of B*V tiles up to 32 (a batch-1 d4 request is one 8-tile forward). "d4" needs height == width."""
        assert num_classes <= 255
        self.device = torch.device(device)
        self.batch, self.H, self.W, self.classes = batch, height, width, num_classes
        self.tta = None
        if tta == "none":
            self.engine = UNetEngine(state_dict, num_classes, batch, height, width, device=self.device, precision=precision)
        else:
            tta_mod.check_shape(tta, height, width)
            engine_batch = tta_mod.TtaChain.engine_batch(tta, batch)
            self.engine = UNetEngine(state_dict, num_classes, engine_batch, height, width, device=self.device, precision=precision)
            self.tta = tta_mod.TtaChain(self.engine, tta, batch, height, width, num_classes, device=self.device)
        self.h_in = torch.empty((batch, height, width, 3), dtype=torch.uint8, pin_memory=True)
        self.d_in = torch.empty((batch, height, width, 3), dtype=torch.uint8, device=self.device)
        self.d_mask = torch.empty((batch, height, width), dtype=torch.uint8, device=self.device)
        self.h_mask = torch.empty((batch, height, width), dtype=torch.uint8, pin_memory=True)
        self.graph = None
        self.graph_error = None
        if use_graph:
            self._capture()

    def _enqueue(self):
        """H2D, forward, argmax, D2H on the current stream (also what the graph records)."""
        self.d_in.copy_(self.h_in, non_blocking=True)
        if self.tta is not None:
            self.tta.argmax(self.d_in, self.d_mask)
            self.h_mask.copy_(self.d_mask, non_blocking=True)
            return
        logits = self.engine.forward(self.d_in)
        _lib.check(_lib.load().rsb_head_argmax(logits.data_ptr(), self.d_mask.data_ptr(), self.batch, self.classes, self.H * self.W,
                                               _lib.current_stream_ptr()), "rsb_head_argmax")
        self.h_mask.copy_(self.d_mask, non_blocking=True)

    def _capture(self):
        # warm up on a side stream first: one-time cudaFuncSetAttribute calls and lazy module loading must not happen
        # while the stream is capturing
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):
                self._enqueue()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(graph):
                self._enqueue()
        except Exception as exc:  # keep serving from the stream (same kernels, launch-bound) and say why
            self.graph_error = "%s: %s" % (type(exc).__name__, exc)
            torch.cuda.synchronize(self.device)
            return
        self.graph = graph

    def run(self):
        """Process what is in `h_in`; returns `h_mask` (pinned, valid until the next call)."""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._enqueue()
        torch.cuda.current_stream(self.device).synchronize()
        return self.h_mask

    def segment_u8(self, tiles):
        """tiles: uint8 [H, W, 3] or [B, H, W, 3] (numpy or torch, host) -> numpy uint8 [H, W] / [B, H, W] class indices."""
        t = tiles.numpy() if torch.is_tensor(tiles) else np.asarray(tiles)
        single = t.ndim == 3
        if single:
            t = t[None]
        assert t.shape == (self.batch, self.H, self.W, 3) and t.dtype == np.uint8, "expected uint8 [B, H, W, 3]"
        self.h_in.numpy()[...] = t  # plain memcpy into the pinned staging buffer
        out = self.run().numpy().copy()
        return out[0] if single else out


class Predictor:
    """Same constructor and `segment(image) -> PIL.Image` contract as robosat/tools/serve.py:135-172."""

    def __init__(self, checkpoint, model, dataset, tta="none"):
        """tta: "none", "flip" or "d4" test-time augmentation of every request (SegmentEngine)"""
        tta_mod.views(tta)  # an unknown mode fails here, not at the first request
        self.tta = tta
        cuda = model["common"]["cuda"]
        assert torch.cuda.is_available() or not cuda, "cuda is available when requested"
        if not cuda:
            raise _lib.RsbError("robosat_b200 serves from an H100 only: set common.cuda = true (there is no CPU path)")
        self.cuda = cuda
        self.device = torch.device("cuda")
        self.checkpoint = checkpoint
        self.model = model
        self.dataset = dataset
        self.num_classes = len(dataset["common"]["classes"])
        chkpt = torch.load(checkpoint, map_location="cpu") if isinstance(checkpoint, str) else checkpoint
        self.state_dict = chkpt["state_dict"]
        self.palette = make_palette(*dataset["common"]["colors"])
        self._engines = {}  # one captured graph per image extent

    def _engine_for(self, height, width):
        eng = self._engines.get((height, width))
        if eng is None:
            eng = self._engines[(height, width)] = SegmentEngine(self.state_dict, self.num_classes, height, width, device=self.device,
                                                                     tta=self.tta)
        return eng

    def segment(self, image):
        rgb = np.asarray(image.convert("RGB"), dtype=np.uint8)  # ConvertImageMode("RGB"), serve.py:154
        mask = self._engine_for(rgb.shape[0], rgb.shape[1]).segment_u8(rgb)
        out = Image.fromarray(mask, mode="P")
        out.putpalette(self.palette)
        return out
