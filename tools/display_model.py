"""Serial model of decode_frames_display's presentation rule (DESIGN 3.18, include/jsmpeg_b200.h), for one stream.

It takes the frames one stream's calls reconstruct, in coded order -- anything with a jsmpeg_b200_frame_t-like info
whose "type" is the picture_coding_type -- and hands them back in presentation order, across call boundaries and
flushes: a B picture is presented at once; an I/P picture first presents the held I/P picture, if any, and is then held
itself (without decode_b: presented at once); flush() presents the held one; drop() forgets it (reset, a seek,
set_index, a call in coded order).  It is the rule of MPEG1Video's displayOrder (jsmpeg_b200/decoder.py,
_render_in_display_order / flush), restricted to the pictures the decoder reconstructs."""
from __future__ import annotations


class DisplayModel:
    def __init__(self, decode_b=True, type_of=lambda frame: frame["type"]):
        self.decode_b = decode_b
        self.type_of = type_of
        self.held = None  # the I/P frame waiting for its successor reference

    def call(self, frames):
        """The frames one call presents, given the frames it reconstructs in coded order."""
        out = []
        for f in frames:
            if self.type_of(f) == 3:
                out.append(f)
                continue
            if self.held is not None:
                out.append(self.held)
                self.held = None
            if self.decode_b:
                self.held = f
            else:
                out.append(f)
        return out

    def flush(self):
        """The frames flush_frames presents: the held one, if any."""
        out = [] if self.held is None else [self.held]
        self.held = None
        return out

    def drop(self):
        self.held = None


def present(frames, calls, decode_b=True, type_of=lambda frame: frame["type"], flush=True):
    """`frames` (coded order) cut into consecutive calls of len(c) frames each for c in `calls` (the last call takes
    what is left), then flushed: the list of each call's presented frames (the flush's last)."""
    model, out, at = DisplayModel(decode_b, type_of), [], 0
    for i, n in enumerate(calls):
        take = frames[at:] if i == len(calls) - 1 else frames[at:at + n]
        at += len(take)
        out.append(model.call(take))
    if flush:
        out.append(model.flush())
    return out
