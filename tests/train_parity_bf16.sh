#!/bin/bash
# BASELINE configs[4] shape (batch 16, 112x112, UIEB-shaped synthetic data): the training loop with the single-pass
# bf16 arithmetic (--train-precision bf16) must follow the loss curve of the same loop with gradients from torch
# autograd (--precision fp32: fp32 CUDA-core forward + torch-graph backward), as tests/train_parity.sh asks of the
# default bf16x3 arithmetic.  Run on the GPU box.
cd "$(dirname "$0")/.."
set -e
EPOCHS=${1:-3}
rm -rf training
python train.py --synthetic --epochs $EPOCHS --seed 0 --train-precision bf16 > /tmp/train_bf16.log 2>&1
python train.py --synthetic --epochs $EPOCHS --seed 0 --precision fp32 > /tmp/train_torch.log 2>&1
grep -E "Train|Val|Total" /tmp/train_bf16.log | sed 's/^/bf16   | /'
grep -E "Train|Val|Total" /tmp/train_torch.log | sed 's/^/torch  | /'
python - <<'PY'
import json
import numpy as np
assert json.load(open("training/0/config.json"))["train_precision"] == "bf16"
a = np.loadtxt("training/0/metrics-train.csv", delimiter=",", skiprows=1).reshape(-1, 5)
b = np.loadtxt("training/1/metrics-train.csv", delimiter=",", skiprows=1).reshape(-1, 5)
rel = np.abs(a - b) / np.maximum(np.abs(b), 1e-9)
print("epoch-wise relative difference of (mse, ssim, psnr, perceptual, loss):")
print(np.array2string(rel[:: max(1, len(rel) // 10)], precision=4))
print("final train metrics bf16:", a[-1], "torch:", b[-1])
assert a[-1, 4] < a[0, 4] * 1.0, "loss did not decrease"
assert rel[: min(len(rel), 5), 4].max() < 0.05, "loss curves diverge in the first epochs"
assert rel[-1, 4] < 0.25, "final losses differ by more than 25 %"
print("train parity (bf16) ok")
PY
rm -rf training
