"""torch.hub surface of the reference (``hubconf.py``) on top of the CUDA engine."""
from __future__ import annotations

import numpy as np
import torch

from .engine import get_engine
from .net import WaterNet

# same artefact the reference fetches (hubconf.py:5); needs network access
DEFAULT_CKPT_URL = "https://www.dropbox.com/s/j8ida1d86hy5tm4/waternet_exported_state_dict-daa0ee.pt?dl=1"


def arr2ten_noeinops(arr, device=None) -> torch.Tensor:
    """uint8 (N)HWC array -> fp32 NCHW tensor in [0,1] on the device (hubconf.py:8-21).

    The division by 255 is a true fp32 division, bit-identical to
    ``torch.from_numpy(arr) / 255``; a 3-D input gains a batch dimension.
    """
    a = np.asarray(arr)
    if a.ndim == 3:
        a = a[None]
    if a.ndim != 4:
        raise ValueError(f"expected (N)HWC, got shape {a.shape}")
    eng = get_engine(device)
    t = torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)
    if t.dtype == torch.uint8 and t.shape[3] == 3:
        return eng.preprocess(t, tensors=True, images=False)["x"]
    # other dtypes / channel counts: true division (a 0-dim tensor divisor; "tensor / python scalar" on CUDA
    # multiplies by a reciprocal and would differ from the reference by an ulp)
    return (t / torch.tensor(255.0, device=t.device)).permute(0, 3, 1, 2)


def ten2arr_noeinops(ten: torch.Tensor) -> np.ndarray:
    """fp32 NCHW tensor -> uint8 NHWC array: clip [0,1], *255, truncate (hubconf.py:24-34)."""
    eng = get_engine(ten.device if ten.is_cuda else None)
    return eng.postprocess(ten.to(eng.device)).cpu().numpy()


def waternet(pretrained: bool = True, device=None, tile=None):
    """Returns ``(preprocess, postprocess, model)`` -- the order ``hubconf.py:96`` returns.

    ``preprocess(rgb_arr)``: HWC (or NHWC) uint8 array -> ``(rgb, wb, he, gc)`` fp32
    (N,3,H,W) tensors on the device (``hubconf.py:85-91``).  ``postprocess(out)``:
    model output -> uint8 NHWC array (``hubconf.py:93-94``).  ``tile`` sets ``model.tile``
    (e.g. 998): the model then runs in overlapping windows, so that images of any size fit; ``"auto"`` runs whole
    images where they fit half the card's memory and windows otherwise, chosen per call (``Engine.auto_tile``).
    """
    eng = get_engine(device)
    model = WaterNet(tile=tile)
    if pretrained is True:
        ckpt = torch.hub.load_state_dict_from_url(DEFAULT_CKPT_URL, progress=False, check_hash=True)
        model.load_state_dict(ckpt)
    model = model.to(eng.device)

    def preprocess(rgb_arr):
        a = np.asarray(rgb_arr)
        if a.ndim == 3:
            a = a[None]
        if a.ndim != 4 or a.shape[3] != 3 or a.dtype != np.uint8:
            raise ValueError(f"preprocess expects an HWC (or NHWC) RGB uint8 array, got {a.dtype} {a.shape}")
        dev_in = torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)
        r = eng.preprocess(dev_in, tensors=True, images=False)
        return r["x"], r["wb"], r["he"], r["gc"]

    def postprocess(model_out):
        return ten2arr_noeinops(model_out)

    return preprocess, postprocess, model
