"""VAE training CLI with the reference's command line (reference vae/train_vae.py:47-161): same flags, same
model-directory naming, same 90/10 split, same early stopping (patience 10 on the validation reconstruction
loss, checkpoint on improvement) -- driving the H100 ConvVAE instead of a TensorFlow session.

What is different on purpose: frames stay uint8 end to end.  The PNGs are decoded once, uploaded once and kept
resident in HBM (38.4 KB/frame); the `/255` (rgb) and `/12` (segmentation class ids, train_vae.py:26-29) scalings
happen inside the first CUDA kernel, and minibatches are gathered on the device.

    python -m carla_ppo_b200.vae.train_vae --dataset /path/to/data --loss_type bce --z_dim 64
"""
from __future__ import annotations

import argparse
import os
import shutil

import numpy as np

from .. import _lib


def read_png_dir(directory: str, channels: int) -> np.ndarray:
    """All ``*.png`` of a directory (os.listdir order, like the reference) as one uint8 array [N,80,160,channels]."""
    from PIL import Image
    frames = []
    for name in os.listdir(directory):
        if os.path.splitext(name)[1] != ".png":
            continue
        img = np.asarray(Image.open(os.path.join(directory, name)))
        frames.append(np.ascontiguousarray(img[:, :, :channels]))
    if not frames:
        raise FileNotFoundError("no .png frames under %s" % directory)
    return np.stack(frames, axis=0)


def split_validation(frames: np.ndarray, val_portion: float = 0.1):
    """First 10 % = validation (reference train_val_split, train_vae.py:41-45)."""
    cut = int(frames.shape[0] * val_portion)
    return frames[cut:], frames[:cut]


MATH_MODES = {"simt": _lib.MATH_SIMT, "3xtf32": _lib.MATH_3XTF32, "tf32": _lib.MATH_TF32}


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="Trains a VAE with RGB images as source and RGB or segmentation images as target")
    p.add_argument("--model_name", type=str, default=None)
    p.add_argument("--dataset", type=str, default="data")
    p.add_argument("--use_segmentation_as_target", type=bool, default=False)
    p.add_argument("--loss_type", type=str, default="bce")
    p.add_argument("--model_type", type=str, default="cnn")
    p.add_argument("--beta", type=int, default=1)
    p.add_argument("--z_dim", type=int, default=64)
    p.add_argument("--learning_rate", type=float, default=1e-4)
    p.add_argument("--lr_decay", type=float, default=1.0)
    p.add_argument("--batch_size", type=int, default=100)
    p.add_argument("--kl_tolerance", type=float, default=0.0)
    p.add_argument("-restart", action="store_true")
    p.add_argument("--max_epochs", type=int, default=0, help="(addition) stop after this many epochs; 0 = early stopping only")
    p.add_argument("--models_root", type=str, default="models", help="(addition) parent directory of the model directories")
    p.add_argument("--math_mode", choices=sorted(MATH_MODES), default="3xtf32",
                   help="(addition) arithmetic of the ConvVAE's conv2-4 / deconv1-3 layers: 3xtf32 (fp32-accurate), "
                        "tf32 (one TF32 tensor-core pass, not fp32-accurate) or simt (fp32 FMA).  The MlpVAE "
                        "(--model_type mlp) runs fp32 SIMT under simt and 3xtf32; tf32 runs its encoder/dense and "
                        "decoder/dense_2 products (forward and gradients) as one TF32 tensor-core pass")
    return p


def default_model_name(args) -> str:
    return "{}_{}_{}_zdim{}_beta{}_kl_tolerance{}_{}".format(
        "seg" if args.use_segmentation_as_target else "rgb", args.loss_type, args.model_type, args.z_dim, args.beta,
        args.kl_tolerance, os.path.splitext(os.path.basename(args.dataset))[0])


def main(argv=None):
    from .models import ConvVAE, MlpVAE, bce_loss, bce_loss_v2, mse_loss
    args = build_parser().parse_args(argv)

    rgb = read_png_dir(os.path.join(args.dataset, "rgb"), 3)
    train_src, val_src = split_validation(rgb)
    if args.use_segmentation_as_target:
        seg = read_png_dir(os.path.join(args.dataset, "segmentation"), 1)
        train_tgt, val_tgt = split_validation(seg)
    else:
        train_tgt, val_tgt = train_src, val_src
    np.random.seed(0)
    if args.model_name is None:
        args.model_name = default_model_name(args)
    for label, arr in (("train_source_images", train_src), ("val_source_images", val_src),
                       ("train_target_images", train_tgt), ("val_target_images", val_tgt)):
        print(label + ".shape", arr.shape)
    print("\nTraining parameters:")
    for k, v in vars(args).items():
        print("  {}: {}".format(k, v))
    print("")

    losses = {"bce": bce_loss, "bce_v2": bce_loss_v2, "mse": mse_loss}
    if args.loss_type not in losses:
        raise Exception("No loss function \"{}\"".format(args.loss_type))
    classes = {"cnn": ConvVAE, "mlp": MlpVAE}
    if args.model_type not in classes:
        raise Exception("No model type \"{}\"".format(args.model_type))
    vae = classes[args.model_type](source_shape=train_src.shape[1:], target_shape=train_tgt.shape[1:], z_dim=args.z_dim,
                                   beta=args.beta, learning_rate=args.learning_rate, lr_decay=args.lr_decay,
                                   kl_tolerance=args.kl_tolerance, loss_fn=losses[args.loss_type],
                                   model_dir=os.path.join(args.models_root, args.model_name))

    restart = args.restart
    if not restart and os.path.isdir(vae.log_dir) and len(os.listdir(vae.log_dir)) > 0:
        answer = input("Model \"{}\" already exists. Do you wish to continue (C) or restart training (R)? ".format(args.model_name))
        if answer.upper() == "R":
            restart = True
        elif answer.upper() != "C":
            raise Exception("There are already log files for model \"{}\". Please delete it or change model_name and try again".format(args.model_name))
    if restart:
        shutil.rmtree(vae.model_dir)
        for d in vae.dirs:
            os.makedirs(d)
    vae.init_session()
    if not restart:
        vae.load_latest_checkpoint()
    _lib.check(_lib.load().cpb_set_math_mode(MATH_MODES[args.math_mode]), "cpb_set_math_mode")

    print("Training")
    best, stale = float("inf"), 0
    while True:
        epoch = vae.get_step_idx()
        if (epoch + 1) % 10 == 0:
            print("Epoch {}".format(epoch + 1))
        val_loss, _ = vae.evaluate(val_src, val_tgt, args.batch_size)
        if val_loss < best:
            best, stale = val_loss, 0
            vae.save()
        else:
            stale += 1
            if stale >= 10:
                print("No improvement in last 10 epochs, stopping")
                break
        if args.max_epochs and epoch >= args.max_epochs:
            break
        vae.train_one_epoch(train_src, train_tgt, args.batch_size)
    return vae


if __name__ == "__main__":
    main()
