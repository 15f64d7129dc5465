"""Score weights on the validation split (same CLI as the reference's score.py).

    python score.py --weights W [--batch-size 16] [--height 112] [--width 112] [--seed S] [--synthetic]
"""
import argparse
from pathlib import Path
from timeit import default_timer as timer

import torch

from waternet.net import WaterNet
from waternet.training_utils import SyntheticUIEB, UIEBDataset
from waternet_b200 import training as T


def main():
    start = timer()
    root = Path(__file__).parent
    torch.manual_seed(0)
    ap = argparse.ArgumentParser()
    ap.add_argument("--weights", type=str, help="Path to the weights to score")
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--height", type=int, default=112)
    ap.add_argument("--width", type=int, default=112)
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--epochs", type=int, default=400, help="accepted for command-line compatibility with the reference's "
                                                            "score.py (:96); scoring runs one validation pass")
    ap.add_argument("--synthetic", action="store_true")
    T.add_perceptual_args(ap)
    T.add_metrics_arg(ap)
    args = ap.parse_args()
    assert args.weights is not None, "No weights specified in --weights!"
    if args.seed is not None:
        torch.manual_seed(args.seed)
    if not torch.cuda.is_available():
        raise SystemExit("score.py needs a CUDA device (H100); waternet_b200 has no CPU path")
    device = torch.device("cuda")
    raw_dir, ref_dir = root / "data/raw-890", root / "data/reference-890"
    if args.synthetic or not raw_dir.exists():
        dataset = SyntheticUIEB(890, args.height, args.width, seed=args.seed or 0)
    else:
        dataset = UIEBDataset(raw_dir, ref_dir, im_height=args.height, im_width=args.width, transform=lambda image, mask: {"image": image, "mask": mask})
    n_val = 90 if len(dataset) >= 180 else max(1, len(dataset) // 10)
    _, val_set = torch.utils.data.random_split(dataset, [len(dataset) - n_val, n_val])
    loader = torch.utils.data.DataLoader(val_set, batch_size=args.batch_size)
    model = WaterNet()
    model.load_state_dict(torch.load(args.weights, map_location="cpu"))
    model.to(device).eval()
    vgg = T.perceptual_model(args).to(device).eval()
    metrics = T.eval_one_epoch(model, loader, vgg, device, native_metrics=args.metrics == "native")
    print("    Val   ||", "   ".join(f"{k}: {v:.03g}" for k, v in metrics.items()))
    print(f"Total time: {timer() - start}s")


if __name__ == "__main__":
    main()
