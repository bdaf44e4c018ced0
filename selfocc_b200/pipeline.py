"""Host-side frame loop for serving the hot path from HOST buffers: the H2D copy of frame k+1 and the D2H copy of
frame k's result overlap the compute of the neighbouring frames (two device input buffers, two side streams).

The reference feeds one frame per iteration from a DataLoader with ``pin_memory`` and copies results back with
``.cpu()`` on the compute stream (eval_depth.py:150-190); serial copies add their full PCIe time to every frame, so the
evaluation loop is written as a 3-stage pipeline instead.  Plumbing only: streams, events, pinned copies."""
import torch


class FramePipeline:
    """``compute(device_inputs) -> out`` runs on the current stream; ``fetch(out)`` names the device tensors to download
    into ``out_host`` (pinned host tensors, same order).

    pipe.submit(host_k, next_host=host_k1) enqueues frame k and starts the upload of frame k+1; the ``host`` of a call
    must be the ``next_host`` of the previous call (or the first frame).  Results of frame k are complete in
    ``out_host`` after ``pipe.drain()`` (or after the next-but-one submit) and a host synchronisation."""

    def __init__(self, compute, fetch, out_host, device, cuda=None):
        self.cuda = cuda if cuda is not None else torch.cuda
        self.compute, self.fetch, self.out_host, self.device = compute, fetch, list(out_host), device
        self.h2d = self.cuda.Stream(device=device)
        self.d2h = self.cuda.Stream(device=device)
        self.bufs = [None, None]      # device input buffers
        self.ready = [None, None]     # event: upload into the buffer has finished
        self.free = [None, None]      # event: the last frame that read the buffer has finished
        self.k = 0

    def _upload(self, slot, host):
        if self.bufs[slot] is None:   # allocated once, on the caller's stream: the block may be recycled memory that work
            self.bufs[slot] = [torch.empty(t.shape, dtype=t.dtype, device=self.device) for t in host]   # already queued there
            self.h2d.wait_stream(self.cuda.current_stream(self.device))                                # still reads
        with self.cuda.stream(self.h2d):
            if self.free[slot] is not None:
                self.h2d.wait_event(self.free[slot])
            for d, s in zip(self.bufs[slot], host):
                d.copy_(s, non_blocking=True)
            ev = self.cuda.Event()
            ev.record(self.h2d)
        self.ready[slot] = ev

    def submit(self, host, next_host=None):
        main = self.cuda.current_stream(self.device)
        slot = self.k & 1
        if self.ready[slot] is None:
            self._upload(slot, host)                      # cold start: this frame's own copy, nothing to overlap with
        main.wait_event(self.ready[slot])
        self.ready[slot] = None
        if next_host is not None:
            self._upload(slot ^ 1, next_host)             # overlaps this frame's compute
        out = self.compute(self.bufs[slot])
        done = self.cuda.Event()
        done.record(main)
        self.free[slot] = done
        srcs = self.fetch(out)
        with self.cuda.stream(self.d2h):
            self.d2h.wait_event(done)
            for h, s in zip(self.out_host, srcs):
                if s.is_cuda:
                    s.record_stream(self.d2h)             # the allocator must not recycle `s` before the copy has run
                h.copy_(s, non_blocking=True)
        self.k += 1
        return out

    def drain(self):
        """Make the current stream wait for every outstanding download."""
        self.cuda.current_stream(self.device).wait_stream(self.d2h)
