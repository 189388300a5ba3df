"""Runs fast3r_b200.views.prepare_views on the CPU with its device calls replaced by recorders (no pixel is computed):
the lib.VIEW_PARAM records of every f3r_view_geometry call, each with the filter its image is resampled with.  Shared by
tests/test_views_plans_cpu.py and tests/test_views_gpu.py."""
import numpy as np
import torch


def record(monkeypatch, calls_fn):
    """Runs calls_fn() (which calls prepare_views(..., device="cpu")) and returns one list of (record, filter) per
    f3r_view_geometry call."""
    from fast3r_b200 import ingest, ops, views
    calls, filts = [], []

    def view_geometry(params, out_pts, out_valid, out_depth):
        calls.append(list(zip(params.copy(), filts[:])))
        filts.clear()

    def resize_crop_rgb8(img_u8, nw, nh, filt, box, out=None):
        filts.append(filt)
        return torch.zeros(3, box[3] - box[1], box[2] - box[0]) if out is None else out

    monkeypatch.setattr(views, "_need_cuda", lambda device: None)
    monkeypatch.setattr(views, "_upload", lambda arr, device: torch.empty(np.shape(arr), device="meta",
                                                                          dtype=torch.from_numpy(np.asarray(arr)[:0]).dtype))
    monkeypatch.setattr(ops, "view_geometry", view_geometry)
    monkeypatch.setattr(ingest, "resize_crop_rgb8", resize_crop_rgb8)
    calls_fn()
    return calls
