"""Train WaterNet (same CLI and artefacts as the reference's train.py; CUDA forward underneath).

    python train.py [--epochs 400] [--batch-size 16] [--height 112] [--width 112] [--weights W] [--seed S]
    python train.py --native-size ...   every image at its own size (ragged batches, WaterNet.forward_many)
    python train.py --ssim-weight 0.5 ...   add 0.5 * (1 - SSIM) to the loss (metrics.ssim_loss)

Writes ``training/<n>/{last.pt, metrics-train.csv, metrics-val.csv, config.json}``.  Without the
UIEB folders (``data/raw-890``, ``data/reference-890``) pass ``--synthetic`` for UIEB-shaped
synthetic pairs (there is no dataset offline).
"""
import argparse
from pathlib import Path
from timeit import default_timer as timer

import torch

from waternet.net import WaterNet
from waternet.training_utils import FlipRotate, GpuBatchLoader, SyntheticUIEB, UIEBDataset
from waternet_b200 import training as T


def main():
    start = timer()
    root = Path(__file__).parent
    torch.manual_seed(0)
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=400, help="(Optional) Num epochs, defaults to 400")
    ap.add_argument("--batch-size", type=int, default=16, help="(Optional) Batch size, defaults to 16")
    ap.add_argument("--height", type=int, default=112, help="(Optional) Image height, defaults to 112")
    ap.add_argument("--width", type=int, default=112, help="(Optional) Image width, defaults to 112")
    ap.add_argument("--weights", type=str, help="(Optional) Starting weights for training")
    ap.add_argument("--seed", type=int, default=None, help="(Optional) Seed for torch, defaults to None")
    ap.add_argument("--synthetic", action="store_true", help="Use UIEB-shaped synthetic pairs (no dataset offline)")
    ap.add_argument("--precision", default="default", choices=["default", "fp32", "bf16x3", "bf16_fp8"])
    ap.add_argument("--train-precision", default="bf16x3", choices=["bf16x3", "bf16"],
                    help="(Optional) Arithmetic of the native training step (WaterNet.train_precision): bf16x3 "
                         "(default, ~1e-5 of fp32) or bf16 (one bf16 tensor-core product, fp32 accumulation, as "
                         "autocast trains convolutions)")
    ap.add_argument("--loader", default="gpu", choices=["gpu", "torch"],
                    help="gpu: batches augmented + preprocessed on the device in one call; torch: the reference's "
                         "per-item DataLoader path")
    ap.add_argument("--grad-tile", type=T.tile_arg, default=None, metavar="N|auto",
                    help="(Optional) Compute the gradients in overlapping windows of N x N output pixels "
                         "(WaterNet.grad_tile): about 12 GB of activations whatever the image and batch size, for "
                         "about 1.5x the arithmetic.  auto: whole images where their activations fit half the card's "
                         "memory, else windows of 998, per batch.  Unset: whole images, ~5.6 KB per pixel")
    ap.add_argument("--native-size", action="store_true",
                    help="(Optional) Train every image at its own size: the dataset without --height/--width (UIEB: "
                         "rounded down to a multiple of 32, as the reference does) and batches of differently sized "
                         "images through WaterNet.forward_many.  With --synthetic: a mix of sizes around "
                         "--height x --width")
    T.add_perceptual_args(ap)
    T.add_metrics_arg(ap)
    T.add_loss_arg(ap)
    args = ap.parse_args()
    if args.native_size and args.loader != "gpu":
        raise SystemExit("--native-size needs --loader gpu (ragged batches are assembled on the device)")
    if args.seed is not None:
        torch.manual_seed(args.seed)
    if not torch.cuda.is_available():
        raise SystemExit("train.py needs a CUDA device (H100); waternet_b200 has no CPU path")
    device = torch.device("cuda")
    print(f"Using device: {device}")
    savedir = T.next_run_dir(root / "training")

    aug = FlipRotate(seed=args.seed) if args.loader == "torch" else None
    raw_dir, ref_dir = root / "data/raw-890", root / "data/reference-890"
    if args.synthetic or not raw_dir.exists():
        if not args.synthetic:
            print(f"{raw_dir} not found: falling back to --synthetic data")
        sizes = None
        if args.native_size:  # a mix of sizes around height x width, multiples of 16, at least 32
            sizes = [(max(32, args.height + dh), max(32, args.width + dw))
                     for dh, dw in ((0, 0), (32, -16), (-16, 32), (16, 16), (-32, 0))]
        dataset = SyntheticUIEB(890, args.height, args.width, seed=args.seed or 0, transform=aug, sizes=sizes)
    else:
        size = (None, None) if args.native_size else (args.height, args.width)
        dataset = UIEBDataset(raw_dir, ref_dir, im_height=size[0], im_width=size[1],
                              transform=aug if aug is not None else (lambda image, mask: {"image": image, "mask": mask}))
    n_val = 90 if len(dataset) >= 180 else max(1, len(dataset) // 10)
    train_set, val_set = torch.utils.data.random_split(dataset, [len(dataset) - n_val, n_val])
    if args.loader == "gpu":
        train_loader = GpuBatchLoader(train_set, args.batch_size, device, augment=True, seed=args.seed,
                                      ragged=args.native_size)
        val_loader = GpuBatchLoader(val_set, args.batch_size, device, augment=True, seed=args.seed,
                                    ragged=args.native_size)
    else:
        train_loader = torch.utils.data.DataLoader(train_set, batch_size=args.batch_size)
        val_loader = torch.utils.data.DataLoader(val_set, batch_size=args.batch_size)

    model = WaterNet(precision=args.precision, train_precision=args.train_precision)
    model.grad_tile = args.grad_tile
    if args.weights is not None:
        model.load_state_dict(torch.load(args.weights, map_location="cpu"))
    model.to(device).train()
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)
    scheduler = torch.optim.lr_scheduler.StepLR(optimizer, step_size=10000, gamma=0.1)
    vgg = T.perceptual_model(args).to(device).eval()

    native_metrics = args.metrics == "native"
    train_hist, val_hist = [], []
    for epoch in range(args.epochs):
        print(f"Epoch {epoch + 1}/{args.epochs}")
        tm = T.train_one_epoch(model, train_loader, optimizer, scheduler, vgg, device, log=print,
                               native_metrics=native_metrics, ssim_weight=args.ssim_weight)
        vm = T.eval_one_epoch(model, val_loader, vgg, device, native_metrics=native_metrics)
        print("    Train ||", "   ".join(f"{k}: {v:.03g}" for k, v in tm.items()))
        print("    Val   ||", "   ".join(f"{k}: {v:.03g}" for k, v in vm.items()))
        train_hist.append(tm)
        val_hist.append(vm)
        savedir.mkdir(parents=True, exist_ok=True)
        torch.save(model.state_dict(), savedir / "last.pt")
    T.save_metrics(savedir, train_hist, val_hist, {
        "epochs": args.epochs, "batch_size": args.batch_size, "im_height": args.height, "im_width": args.width,
        "weights": args.weights, "native_size": args.native_size, "grad_tile": args.grad_tile,
        "train_precision": args.train_precision, **T.perceptual_config(args), **T.metrics_config(args),
        **T.loss_config(args)})
    print(f"Metrics and weights saved to {savedir}")
    print(f"Total time: {timer() - start}s")


if __name__ == "__main__":
    main()
