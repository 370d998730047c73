"""Tile-batch inference API: the H100 replacement for the body of the `rs predict` batch loop.

Reference loop body (robosat/tools/predict.py:81-103):
    images.to(device) -> net(images) -> softmax(outputs, 1).cpu().numpy() -> unbuffer (crop overlap)
    -> np.digitize(foreground, linspace(0, 1, 256)).astype(uint8)
Here one call takes a HOST batch (raw uint8 RGB tiles, or the reference's normalised fp32 NCHW tensors),
copies it to the device from pinned memory, runs the U-Net plan and the fused softmax/crop/quantise head on
the device and copies back only the uint8 foreground bins (1 byte per pixel instead of 8).
"""

import torch

from robosat_b200 import _lib
from robosat_b200.engine import UNetEngine
from robosat_b200.tta import TtaChain


class TilePredictor:
    def __init__(self, state_dict, num_classes, batch, size, overlap=0, device="cuda", depth=2, precision=None, use_graph=False, tta="none"):
        """size: net input extent (tile_size + 2*overlap, predict.py:75); depth: in-flight batches for copy/compute overlap.
        use_graph=True captures the 60 launches of (network + head) once per slot into a CUDA graph and replays it: ONE driver
        call per batch instead of 60 ctypes launches. The kernels and results are identical; it matters when the launching thread
        shares the interpreter with decode / encode / consumer threads (`rs predict`: the 60 launches took 5 ms per batch there and
        the device ran ahead of them). If capture fails the predictor keeps launching kernel by kernel (`graph_error` says why).
        tta="flip" | "d4": the bins are those of the mean probability over 2 | 8 dihedral views of each tile (robosat_b200/tta.py);
        the network then runs on an engine of B*V/P tiles, P passes per batch, and the graph records the whole chain."""
        self.device = torch.device(device)
        self.batch, self.size, self.overlap, self.classes = batch, size, overlap, num_classes
        self.tta = None
        if tta == "none":
            self.engine = UNetEngine(state_dict, num_classes, batch, size, size, device=self.device, precision=precision)
        else:
            engine_batch = TtaChain.engine_batch(tta, batch)
            self.engine = UNetEngine(state_dict, num_classes, engine_batch, size, size, device=self.device, precision=precision)
            self.tta = TtaChain(self.engine, tta, batch, size, size, num_classes, overlap, device=self.device)
        self.out_size = size - 2 * overlap
        self.depth = depth
        self._slots = []
        for _ in range(depth):
            self._slots.append({
                "h_in": torch.empty((batch, size, size, 3), dtype=torch.uint8, pin_memory=True),
                "d_in": torch.empty((batch, size, size, 3), dtype=torch.uint8, device=self.device),
                "d_q": torch.empty((batch, self.out_size, self.out_size), dtype=torch.uint8, device=self.device),
                "h_q": torch.empty((batch, self.out_size, self.out_size), dtype=torch.uint8, pin_memory=True),
                "done": torch.cuda.Event(),
                "loaded": torch.cuda.Event(),
                "consumed": torch.cuda.Event(),
                "computed": torch.cuda.Event(),
            })
        self._copy_in = torch.cuda.Stream(device=self.device)
        self._copy_out = torch.cuda.Stream(device=self.device)
        self._next = 0
        self._pending = []
        self.h2d_bytes = batch * size * size * 3
        self.d2h_bytes = batch * self.out_size * self.out_size
        self.graph_error = None
        if use_graph and num_classes == 2:
            self._capture_graphs()

    def _compute(self, slot):
        """network + head of one slot on the current stream: a graph replay if one was captured, else 60 launches"""
        g = slot.get("graph")
        if g is not None:
            g.replay()
        else:
            self._enqueue(slot)

    def _enqueue(self, slot):
        if self.tta is not None:
            self.tta.quantize(slot["d_in"], slot["d_q"])
        else:
            self.quantize(self.engine.forward(slot["d_in"]), slot["d_q"])

    def _capture_graphs(self):
        # warm up on a side stream first (one-time cudaFuncSetAttribute calls must not happen while a stream is capturing)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for slot in self._slots:
                slot["d_in"].zero_()
                self._enqueue(slot)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        try:
            for slot in self._slots:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    self._enqueue(slot)
                slot["graph"] = graph
        except Exception as exc:  # same kernels, launched one by one
            self.graph_error = "%s: %s" % (type(exc).__name__, exc)
            for slot in self._slots:
                slot.pop("graph", None)
            torch.cuda.synchronize(self.device)

    # ------------------------------------------------------------------ device-resident pieces
    def logits(self, x_dev):
        """fp32 NCHW logits (engine-owned buffer) for a device batch: uint8 NHWC raw or fp32 NCHW normalised."""
        return self.engine.forward(x_dev)

    def quantize(self, logits, out_u8, probs=None):
        """softmax -> foreground -> crop overlap -> np.digitize bins (predict.py:87-103), binary models only."""
        assert self.classes == 2, "single channel requires binary model"  # predict.py:98
        lib = _lib.load()
        _lib.check(lib.rsb_head_quantize(logits.data_ptr(), out_u8.data_ptr(), probs.data_ptr() if probs is not None else None,
                                         self.batch, self.size, self.size, self.overlap, _lib.current_stream_ptr()), "rsb_head_quantize")
        return out_u8

    def num_launches(self):
        if self.tta is not None:
            return self.tta.num_launches()
        return self.engine.num_launches() + 1

    # ------------------------------------------------------------------ host -> host
    def predict_u8(self, tiles_u8_host):
        """Blocking: host uint8 [B, S, S, 3] -> host uint8 [B, S-2o, S-2o] quantised foreground probability."""
        self.submit(tiles_u8_host)
        return self.collect()

    def submit(self, tiles_u8_host):
        """Enqueue one batch (H2D copy, forward, head, D2H copy) without waiting for it.

        Copies run on their own streams, ordered by per-slot events only, so the H2D of batch i+1 and the D2H of
        batch i-1 overlap the forward pass of batch i."""
        slot = self._slots[self._next % self.depth]
        self._next += 1
        main = torch.cuda.current_stream(self.device)
        if slot.get("busy"):
            slot["done"].synchronize()  # host side: the pinned buffers of this slot are free again
        src = tiles_u8_host
        if not src.is_pinned():
            slot["h_in"].copy_(src)  # pageable memory: stage through the slot's pinned buffer
            src = slot["h_in"]
        with torch.cuda.stream(self._copy_in):
            if slot.get("busy"):
                self._copy_in.wait_event(slot["consumed"])  # previous forward that read d_in has finished
            slot["d_in"].copy_(src, non_blocking=True)  # pinned source: DMA straight from the caller's buffer
            slot["loaded"].record(self._copy_in)
        main.wait_event(slot["loaded"])
        self._compute(slot)
        slot["consumed"].record(main)
        slot["computed"].record(main)
        with torch.cuda.stream(self._copy_out):
            self._copy_out.wait_event(slot["computed"])
            slot["h_q"].copy_(slot["d_q"], non_blocking=True)
            slot["done"].record(self._copy_out)
        slot["busy"] = True
        self._pending.append(slot)

    def device_input(self):
        """The device input buffer the next `submit_device` will read: fill it on the current stream (e.g. with
        `HaloStitcher.stitch`) instead of copying a host batch."""
        slot = self._slots[self._next % self.depth]
        if slot.get("busy"):
            # the forward pass that last read this buffer must be done before new kernels overwrite it
            torch.cuda.current_stream(self.device).wait_event(slot["consumed"])
        return slot["d_in"]

    def submit_device(self):
        """`submit` for a batch that is already in `device_input()`: forward, head, D2H -- no host-to-device copy."""
        slot = self._slots[self._next % self.depth]
        self._next += 1
        main = torch.cuda.current_stream(self.device)
        if slot.get("busy"):
            slot["done"].synchronize()
        self._compute(slot)
        slot["consumed"].record(main)
        slot["computed"].record(main)
        with torch.cuda.stream(self._copy_out):
            self._copy_out.wait_event(slot["computed"])
            slot["h_q"].copy_(slot["d_q"], non_blocking=True)
            slot["done"].record(self._copy_out)
        slot["busy"] = True
        self._pending.append(slot)

    def pinned_input(self):
        """The pinned staging buffer the next `submit` will use (fill it in place to skip one host copy)."""
        return self._slots[self._next % self.depth]["h_in"]

    def collect(self, poll=False):
        """Wait for the oldest submitted batch and return its pinned host result (valid until `depth` more submits).
        poll=True: wait by polling the event with short sleeps instead of a blocking synchronize -- for a consumer THREAD, so that
        the wait can never keep the interpreter away from the thread that launches the next batch."""
        slot = self._pending.pop(0)
        if poll:
            import time

            while not slot["done"].query():
                time.sleep(0.0002)
        else:
            slot["done"].synchronize()
        return slot["h_q"]
