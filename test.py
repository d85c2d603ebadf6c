#!/usr/bin/env python
"""Inference entry point with the reference's CLI (reference test.py:15-69):
loads <checkpoints_dir>/<name>/<which_epoch>_net_{G,Corr}.pth (reference checkpoints load unchanged)
and writes label | exemplar | warp | output grids, or with --save_per_img one output image per input.
Every batch goes through Pix2PixModel.run_inference (the forward replayed from one CUDA graph on a GPU)."""
import os
import sys

import torch
import torchvision.utils as vutils

from cocosnet_b200 import data as cdata
from cocosnet_b200.options import TestOptions
from cocosnet_b200.pix2pix_model import Pix2PixModel


def per_image_name(path, dataset_mode):
    """File name of one output image (reference test.py:43-46): the input's base name, or for deepfashion its path
    below Dataset/DeepFashion/ with '/' turned into '_'.  The extension picks the format (ade20k: JPEG)."""
    if dataset_mode == "deepfashion":
        return path.split("Dataset/DeepFashion/")[-1].replace("/", "_")
    return os.path.basename(path)


def main():
    opt = TestOptions().parse(sys.argv[1:])
    torch.manual_seed(0)
    dataloader = cdata.create_dataloader(opt)
    model = Pix2PixModel(opt)
    if len(opt.gpu_ids) > 0:
        model.cuda()
    model.eval()
    output_root = os.path.join(os.path.dirname(opt.checkpoints_dir), "output")
    save_root = os.path.join(output_root, "test_per_img" if opt.save_per_img else "", opt.name)
    os.makedirs(save_root, exist_ok=True)
    for i, data_i in enumerate(dataloader):
        if i * opt.batchSize >= opt.how_many:
            break
        out = model.run_inference(data_i)
        if opt.save_per_img:
            imgs = (out["fake_image"].cpu() + 1) / 2
            for j in range(imgs.shape[0]):
                vutils.save_image(imgs[j:j + 1], os.path.join(save_root, per_image_name(data_i["path"][j],
                                                                                        opt.dataset_mode)),
                                  nrow=1, padding=0, normalize=False)
            continue
        imgs = torch.cat((data_i["ref"], out["warp_out"].cpu(), out["fake_image"].cpu()), 0)
        vutils.save_image(imgs, os.path.join(save_root, "%d.png" % i), nrow=data_i["ref"].shape[0], padding=0,
                          normalize=True)
    print("wrote", save_root)


if __name__ == "__main__":
    main()
