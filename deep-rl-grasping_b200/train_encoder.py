"""Command line of the reference's encoder training script (manipulation_main/training/train_encoder.py:30-65), with the
model on the GPU (``b200grasp.encoders.SimpleAutoEncoder``).

    python -m b200grasp.train_encoder <model_dir> train --config <config.yaml> [--train_precision {fp32,bf16x3}]
    python -m b200grasp.train_encoder <model_dir> test [--train_precision {fp32,bf16x3}]

``--train_precision`` picks the arithmetic of the training handle (``SimpleAutoEncoder(train_precision=...)``): fp32 (the
default) or bf16x3 (the tensor-core engine).

The dataset is the reference's pickle ``{'train' | 'test': {'rgb', 'depth', 'masks'}}`` at the config's ``data_path``.
``plot_history`` and ``visualize`` (matplotlib) are not provided.
"""
from __future__ import annotations

import argparse
import os
import pickle

import numpy as np
import yaml

from . import encoders


def _load_data_set(data_path, test):
    with open(os.path.expanduser(data_path), "rb") as f:
        dataset = pickle.load(f)
    return dataset["test"] if test else dataset["train"]


def _preprocess_depth(data_set):
    """train_encoder.py:19-27: zero the flat surface (mask == 0) and the gripper (mask == max)."""
    depth_imgs = data_set["depth"]
    masks = data_set["masks"]
    for i in range(depth_imgs.shape[0]):
        img, mask = depth_imgs[i].squeeze(), masks[i].squeeze()
        img[mask == 0] = 0.
        img[mask == np.max(mask)] = 0.
        depth_imgs[i, :, :, 0] = img
    return depth_imgs


def _load_yaml(path):
    with open(os.path.expanduser(path)) as f:
        return yaml.safe_load(f)


def train(args):
    config = _load_yaml(args.config)
    model_dir = os.path.expanduser(args.model_dir)
    os.makedirs(model_dir, exist_ok=True)
    model = encoders.SimpleAutoEncoder(config, seed=args.seed, train_precision=args.train_precision)
    with open(os.path.join(model_dir, "config.yaml"), "w") as f:
        yaml.safe_dump(config, f, default_flow_style=False)
    train_imgs = _preprocess_depth(_load_data_set(config["data_path"], test=False))
    return model.train(train_imgs, train_imgs, config["batch_size"], config["epochs"], model_dir)


def test(args):
    config = _load_yaml(os.path.join(os.path.expanduser(args.model_dir), "config.yaml"))
    model = encoders.SimpleAutoEncoder(config, train_precision=args.train_precision)
    model.load_weights(args.model_dir)
    test_imgs = _preprocess_depth(_load_data_set(config["data_path"], test=True))
    loss = model.test(test_imgs, test_imgs)
    print("Test loss: {}".format(loss))
    return loss


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("model_dir", type=str)
    subparsers = parser.add_subparsers()
    train_parser = subparsers.add_parser("train")
    train_parser.add_argument("--config", type=str, required=True)
    train_parser.add_argument("--seed", type=int, default=None, help="seeds the initial weights and the shuffling")
    train_parser.set_defaults(func=train)
    test_parser = subparsers.add_parser("test")
    test_parser.set_defaults(func=test)
    for p in (train_parser, test_parser):
        p.add_argument("--train_precision", choices=sorted(encoders.ENCODER_PRECISIONS), default="fp32",
                       help="arithmetic of the training handle: fp32 (CUDA cores) or bf16x3 (tensor cores)")
    args = parser.parse_args(argv)
    if not hasattr(args, "func"):
        parser.error("choose a sub-command: train or test")
    return args.func(args)


if __name__ == "__main__":
    main()
