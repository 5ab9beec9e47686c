"""Per-phase device timing of a training step with CUDA events on the launching stream (no host synchronisation inside
the step).  The trainer and the task call ``mark(name)`` at phase boundaries when a timer is attached; the time between
two consecutive marks is attributed to the LATER mark's name.  Used by bench.py to say what the multi-GPU step spends
outside the GEMMs (gather, scoring, exposed gradient all-reduce wait, optimizer)."""
import collections

import torch


class PhaseTimer:
    def __init__(self):
        self.steps = []
        self.cur = None

    def begin(self):
        self.cur = []
        self.mark("begin")

    def mark(self, name):
        if self.cur is None:
            return
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self.cur.append((name, ev))

    def end(self):
        if self.cur is not None:
            self.steps.append(self.cur)
        self.cur = None

    def summary(self):
        """{phase: mean ms per step} in first-seen order (synchronises)."""
        torch.cuda.synchronize()
        tot = collections.OrderedDict()
        for marks in self.steps:
            for (_, a), (name, b) in zip(marks[:-1], marks[1:]):
                tot[name] = tot.get(name, 0.0) + a.elapsed_time(b)
        n = max(1, len(self.steps))
        return {k: v / n for k, v in tot.items()}
