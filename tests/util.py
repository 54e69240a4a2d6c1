"""Shared helpers for the parity tests (seeded synthetic inputs, comparison)."""
import time

import numpy as np


def rng(seed=1701):     # seed mirrors the reference's GradientChecker (test_gradient_check_util.hpp:25)
    return np.random.default_rng(seed)


def smooth_images(r, n, h, w, shift=(1.7, -2.3)):
    """Two BGR frames with integer values 0..255 as scripts/run-flownet.py:30-35 feeds them: low-pass noise,
    second frame = first shifted by a sub-pixel offset plus noise."""
    import scipy.ndimage as ndi
    base = r.standard_normal((n, 3, h + 16, w + 16))
    base = ndi.gaussian_filter(base, sigma=(0, 0, 3, 3))
    base = (base - base.min()) / (base.max() - base.min())
    a = base[:, :, 8:8 + h, 8:8 + w]
    b = ndi.shift(base, (0, 0, shift[1], shift[0]), order=1, mode="nearest")[:, :, 8:8 + h, 8:8 + w]
    b = b + 0.01 * r.standard_normal(b.shape)
    to8 = lambda x: np.clip(np.round(x * 255), 0, 255).astype(np.float32)
    return to8(a), to8(b)


def maxabs(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    nan_a, nan_b = np.isnan(a), np.isnan(b)
    assert (nan_a == nan_b).all(), "NaN pattern differs"
    d = np.abs(np.where(nan_a, 0, a) - np.where(nan_b, 0, b))
    return float(d.max()) if d.size else 0.0


def kernels_per_case(runs):
    """Names of the kernels each of runs launches, from one profiler session.  Every run sits in a window of its own between
    synchronisations, 2 ms from the next.  A kernel belongs to the window of its launch call (the profiler gives both the
    same correlation id), else to the window its start falls in or is nearest to (a warm-up run of the first case before
    the windows lands in that case's).  A session in which some window has no kernel at all (the profiler now and then
    drops device activity) is taken again; the windows' own annotations on the device timeline do not count as kernels."""
    import torch
    cpu, cuda = torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[cpu, cuda]) as prof:
            runs[0]()                                   # the session's first kernels can go unrecorded
            torch.cuda.synchronize()
            time.sleep(0.002)
            for i, run in enumerate(runs):
                with torch.profiler.record_function("ew_case_%d" % i):
                    run()
                    torch.cuda.synchronize()
                time.sleep(0.002)
        events = prof.events()
        win = {int(e.name[8:]): e.time_range for e in events if e.name.startswith("ew_case_")}

        def window(t):
            return min(win, key=lambda i: max(win[i].start - t, t - win[i].end, 0))

        launch = {e.id: window(e.time_range.start) for e in events
                  if e.device_type == torch.autograd.DeviceType.CPU and "LaunchKernel" in e.name}
        names = [set() for _ in runs]
        for e in events:     # the device timeline also carries the ew_case_ ranges: not kernels, so a window with one only is empty
            if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("ew_case_"):
                names[launch.get(e.id, window(e.time_range.start))].add(e.name)
        if all(names):
            break
    return names
