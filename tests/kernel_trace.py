"""Which CUDA kernels a call launched, read from torch.profiler, with a control against lost records.

Late in a long test process (the whole GPU suite on an H100), profiler sessions come back without kernel records, often
several in a row; a session's first and last kernels are the ones most often missing, and idle time at both ends of the
session makes losses rarer without ending them.  So an empty answer does not show that a kernel did not run.  Every
session therefore idles on the host at both ends, and brackets the call with
two marker kernels (torch.cuda._sleep -> ATen's spin_kernel) on the same stream, the first before the call, the second
after its work has finished.  Only a session with both markers recorded is used: it recorded everything in between, the
call's kernels included.  Otherwise the call runs again in a new session with longer idle ends."""
import time

import torch

MARKER = "spin_kernel"
DISCARDED = [0]        # sessions discarded in this process


def launched_kernels(fn, keep, sessions=12, pad=0.05):
    """(fn()'s result, {names of the kernels it launched for which keep(name) holds}) from the first session that
    recorded both markers.  Lost sessions come in runs (in the full GPU suite about half the sessions of its last files
    lose their records, at times five in a row), hence the number of sessions."""
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(sessions):
        idle = min(pad * 2 ** attempt, 0.4)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(idle)
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            time.sleep(idle)
        events = prof.key_averages()
        if sum(e.count for e in events if MARKER in e.key) >= 2:
            return out, {e.key for e in events if keep(e.key) and MARKER not in e.key}
        DISCARDED[0] += 1
    raise AssertionError("torch.profiler lost the marker records of %d sessions in a row" % sessions)


def launched_kernels_each(fns, keep, sessions=12, pad=0.05):
    """[{names of the kernels fns[i]() launched for which keep(name) holds} for each i] from ONE profiler session: a
    marker kernel before each call and after the last, the device records ordered by start time and cut at the markers.
    A process that opens many sessions makes later sessions lose their records more often, so a test that needs the
    kernels of many calls asks for them here, once.  Only a session with all len(fns) + 1 markers recorded is used;
    otherwise every fn runs again in a new session with longer idle ends, so each fn must be callable repeatedly."""
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(sessions):
        idle = min(pad * 2 ** attempt, 0.4)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(idle)
            for fn in fns:
                torch.cuda._sleep(1000)
                torch.cuda.synchronize()
                fn()
                torch.cuda.synchronize()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            time.sleep(idle)
        events = sorted((e.start_ns(), e.name()) for e in prof.profiler.kineto_results.events()
                        if e.device_type() == torch.autograd.DeviceType.CUDA)
        if sum(MARKER in name for _, name in events) == len(fns) + 1:
            out, cur = [], None
            for _, name in events:
                if MARKER in name:
                    if cur is not None:
                        out.append(cur)
                    cur = set()
                elif cur is not None and keep(name):
                    cur.add(name)
            return out
        DISCARDED[0] += 1
    raise AssertionError("torch.profiler lost the marker records of %d sessions in a row" % sessions)
