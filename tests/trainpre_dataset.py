"""TEST INFRASTRUCTURE ONLY -- a PNG dataset with the item protocol of the reference's tools/datasets/BaseDataset.py in 'train' mode,
so that the end-to-end loader case of tests/golden/trainpre.npz also runs where no copy of the reference is available.

What the golden batches depend on, and what this class therefore does in the same order: the file list `<root>/train.txt` is
shuffled with Python's global `random` when the dataset is built; an item reads the image with cv2 (BGR) and flips it to RGB, reads
the label as grayscale, calls the preprocess, and returns data (float) / label (long) / fn (the label's file stem) / n, with the
preprocess's extra_dict merged in."""
import os
import random

import cv2
import numpy as np
import torch
import torch.utils.data as tud


class BaseDataset(tud.Dataset):
    def __init__(self, root, preprocess):
        with open(os.path.join(root, "train.txt")) as f:
            files = f.readlines()
        random.shuffle(files)
        self.root, self.preprocess = root, preprocess
        self.names = [line.strip().split(" ") for line in files]

    def __len__(self):
        return len(self.names)

    def __getitem__(self, i):
        img_name, gt_name = self.names[i]
        img = cv2.imread(os.path.join(self.root, img_name), cv2.IMREAD_COLOR)[:, :, ::-1]
        gt = cv2.imread(os.path.join(self.root, gt_name), cv2.IMREAD_GRAYSCALE)
        img, gt, extra = self.preprocess(img, gt)
        out = dict(data=torch.from_numpy(np.ascontiguousarray(img)).float(), label=torch.from_numpy(np.ascontiguousarray(gt)).long(),
                   fn=gt_name.split("/")[-1].split(".")[0], n=len(self.names))
        for k, v in (extra or {}).items():
            out[k] = torch.from_numpy(np.ascontiguousarray(v))
        return out


def train_loader(root, preprocess, batch, workers):
    """the DataLoader the reference's get_train_loader builds (shuffled, drop_last, pinned) over this dataset"""
    return tud.DataLoader(BaseDataset(root, preprocess), batch_size=batch, num_workers=workers, drop_last=True, shuffle=True,
                          pin_memory=True)
