"""Frames in flight.

One forward of the path is an encoder that fills the GPU (persistent tensor-core kernels) followed by a decoder that
is a dependent chain of ~90 small kernels on 200 query rows, during which most SMs idle.  Frames are independent in
eval mode, so a serving loop can keep `depth` frames in flight on `depth` CUDA streams: the decoder of frame i then
overlaps the encoder of frame i+1.  Every stream has its own CUDA graph and output buffers (graph.GraphCache keys on
the stream), results are bit-identical to the single-stream path; only the scheduling differs.
"""
import torch

from . import _lib


class FramePipeline:
    def __init__(self, neck, head, depth=3, device=None, tc_sms=140):
        """depth: frames in flight.
        tc_sms: with depth > 1 the persistent tensor-core grids are capped at this many CTAs so that the other frames'
        small decoder kernels always find a free SM (process-wide setting of libdi_b200; 0 = leave as is)."""
        self.neck, self.head, self.depth = neck, head, depth
        self.streams = [torch.cuda.Stream(device=device) for _ in range(depth)]
        self.count = 0
        if depth > 1 and tc_sms:
            L = _lib.lib()
            _lib.check(L.di_tc_set_sm_limit(int(tc_sms)), 'di_tc_set_sm_limit')

    def submit(self, frame, wait_event=None, stream_index=None):
        """frame: dict(img_feats, pts_feats, img_metas, pts_metas) of device tensors.  Returns (out, done_event,
        stream): `out` (the decoder's merged dict) lives in that stream's graph buffers and is valid until the next
        submit on the same stream (i.e. `depth` submits later) -- consume it on `stream` or after `done_event`."""
        i = self.count % self.depth if stream_index is None else stream_index
        self.count += 1
        s = self.streams[i]
        s.wait_stream(torch.cuda.current_stream())          # inputs produced on the caller's stream
        with torch.cuda.stream(s):
            if wait_event is not None:
                s.wait_event(wait_event)
            img, pts = self.neck(frame['img_feats'], frame['pts_feats'], frame['img_metas'], frame['pts_metas'])
            out = self.head(pts, img, frame['img_metas'])[0][0]
            done = torch.cuda.Event()
            done.record(s)
        return out, done, s

    def warm(self, frame, rounds=3):
        """Run `rounds` forwards per stream so that every stream owns its captured graphs (the encoder graph is
        captured on the 2nd sighting of a signature, the decoder's on the sighting after that)."""
        for _ in range(rounds):
            for i in range(self.depth):
                self.submit(frame, stream_index=i)
        self.join()

    def join(self):
        cur = torch.cuda.current_stream()
        for s in self.streams:
            cur.wait_stream(s)
