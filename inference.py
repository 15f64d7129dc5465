"""Enhance images / videos (same CLI and output layout as the reference's inference.py).

    python inference.py --source <image|video|directory> [--weights W] [--name NAME] [--show-split]
                        [--tile N|auto] [--batch N]

Every frame goes uint8 -> GPU (preprocess, gated-fusion forward, uint8 postprocess) -> uint8
through ``waternet_b200.api.Enhancer``; video frames are processed in small batches.  File and
codec I/O stays with OpenCV.  Results land in ``output/<NAME or next number>/``.
"""
import argparse
import os
from pathlib import Path

import numpy as np
import torch

from waternet.net import WaterNet
from waternet_b200.api import Enhancer
from waternet_b200.hub import DEFAULT_CKPT_URL
from waternet_b200.training import next_run_dir, tile_arg

ROOT = Path(__file__).parent.resolve()
DEFAULT_CKPT = "waternet_exported_state_dict-daa0ee.pt"
VID_SUFFIXES = [".mp4", ".mpeg", ".avi"]
IM_SUFFIXES = [".bmp", ".jpg", ".jpeg", ".png", ".gif"]
VIDEO_BATCH = 4


def load_model(weights):
    model = WaterNet()
    if weights is None:
        print(f"No weights specified in --weights, using default: {DEFAULT_CKPT}")
        path = ROOT / DEFAULT_CKPT
        if path.exists():
            sd = torch.load(path, map_location="cpu")
        else:  # needs network access, like the reference
            sd = torch.hub.load_state_dict_from_url(DEFAULT_CKPT_URL, progress=False, map_location="cpu",
                                                    model_dir=ROOT, check_hash=True)
    else:
        sd = torch.load(weights, map_location="cpu")
    model.load_state_dict(sd)
    return model.cuda().eval()


def split_view(cv2, before_bgr, after_bgr):
    """Left half original, right half enhanced, with Before/After captions."""
    canvas = np.zeros_like(before_bgr)
    half = after_bgr.shape[1] // 2
    canvas[:, :half] = before_bgr[:, :half]
    canvas[:, half:] = after_bgr[:, half:]
    for text, x in (("Before", 50), ("After", half + 50)):
        cv2.putText(img=canvas, text=text, org=(x, 50), fontFace=cv2.FONT_HERSHEY_DUPLEX, fontScale=1,
                    color=(255, 255, 255), thickness=2)
    return canvas


def run_image(cv2, enhancer, path, savedir, show_split):
    bgr = cv2.imread(os.fspath(path))
    rgb = np.ascontiguousarray(bgr[..., ::-1])
    out_bgr = np.ascontiguousarray(enhancer(rgb)[..., ::-1])
    savedir.mkdir(parents=True, exist_ok=True)
    cv2.imwrite(os.fspath(savedir / path.name), split_view(cv2, bgr, out_bgr) if show_split else out_bgr)


def run_images(cv2, enhancer, paths, savedir, show_split):
    """Several still images of their own sizes in one ragged call (``--batch``); written as run_image writes them."""
    bgrs = [cv2.imread(os.fspath(p)) for p in paths]
    outs = enhancer.enhance_many([np.ascontiguousarray(b[..., ::-1]) for b in bgrs])
    savedir.mkdir(parents=True, exist_ok=True)
    for path, bgr, out in zip(paths, bgrs, outs):
        out_bgr = np.ascontiguousarray(out[..., ::-1])
        cv2.imwrite(os.fspath(savedir / path.name), split_view(cv2, bgr, out_bgr) if show_split else out_bgr)


def run_video(cv2, enhancer, path, savedir, show_split):
    cap = cv2.VideoCapture(os.fspath(path))
    fps = int(cap.get(cv2.CAP_PROP_FPS))
    width, height = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    total = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
    print(f"frame_width={width}, frame_height={height}")
    savedir.mkdir(parents=True, exist_ok=True)
    writer = cv2.VideoWriter(os.fspath(savedir / (path.stem + ".mp4")), cv2.VideoWriter.fourcc(*"avc1"), fps,
                             (width, height))
    print(f"Working on {path.name} with {total} frames")
    done, pending = 0, []

    def flush():
        nonlocal done
        if not pending:
            return
        rgb = np.stack([f[..., ::-1] for f in pending])
        out = enhancer(rgb)
        for before, after in zip(pending, out):
            after_bgr = np.ascontiguousarray(after[..., ::-1])
            writer.write(split_view(cv2, before, after_bgr) if show_split else after_bgr)
            done += 1
            if done % 50 == 0:
                print(f"Processed {done} frames")
        pending.clear()

    while True:
        ok, bgr = cap.read()
        if not ok:
            break
        pending.append(bgr)
        if len(pending) == VIDEO_BATCH:
            flush()
    flush()
    cap.release()
    writer.release()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--source", type=str, help="Path to input image/video/directory (bmp, jpg, jpeg, png, gif; "
                                               "mp4, mpeg, avi)")
    ap.add_argument("--weights", type=str, help=f"(Optional) Path to model weights, defaults to {DEFAULT_CKPT}")
    ap.add_argument("--name", type=str, help="(Optional) Subfolder name to save under `./output`.")
    ap.add_argument("--show-split", action="store_true", default=False,
                    help="(Optional) Left/right of output is original/processed, with a before/after watermark.")
    ap.add_argument("--tile", type=tile_arg, default=None, metavar="N|auto",
                    help="(Optional) Compute each image in overlapping tiles of at most N x N output pixels: the same "
                         "result with GPU memory that does not grow with the image size (e.g. 998 for large photos).  "
                         "auto: whole images where they fit half the card's memory, else tiles of 998, per call.")
    ap.add_argument("--batch", type=int, default=1,
                    help="(Optional) Enhance the still images of a directory N at a time, each at its own size, in "
                         "one GPU call per group (the same result; --tile sets the tile of that call).")
    args = ap.parse_args()
    assert args.batch >= 1, "--batch must be at least 1"
    assert args.source is not None, "No input image/video specified in --source!"
    if not torch.cuda.is_available():
        raise SystemExit("inference.py needs a CUDA device (H100); waternet_b200 has no CPU path")
    print("Using device: cuda")
    import cv2  # file / codec I/O only

    enhancer = Enhancer(load_model(args.weights), tile=args.tile)
    source = Path(args.source)
    assert source.exists(), f"{args.source} does not exist!"
    files = [source] if not source.is_dir() else [
        p for p in sorted(source.glob("*")) if p.suffix.lower() in VID_SUFFIXES + IM_SUFFIXES]
    print(f"Total images/videos: {len(files)}")
    outdir = ROOT / "output"
    outdir.mkdir(exist_ok=True)
    savedir = outdir / args.name if args.name is not None else next_run_dir(outdir)
    pending = []  # still images waiting for a group of --batch
    for f in files:
        if f.suffix.lower() in IM_SUFFIXES:
            if args.batch == 1:
                run_image(cv2, enhancer, f, savedir, args.show_split)
                continue
            pending.append(f)
            if len(pending) == args.batch:
                run_images(cv2, enhancer, pending, savedir, args.show_split)
                pending = []
        elif f.suffix.lower() in VID_SUFFIXES:
            run_video(cv2, enhancer, f, savedir, args.show_split)
    if pending:
        run_images(cv2, enhancer, pending, savedir, args.show_split)
    print(f"Saved output to {savedir}!")


if __name__ == "__main__":
    main()
