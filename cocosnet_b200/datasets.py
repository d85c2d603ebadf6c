"""Readers for the real ADE20k, CelebA-HQ and DeepFashion datasets.

For the same state of Python's `random` every reader returns the same batch dict, bit for bit, as the reference's
dataset classes (data/base_dataset.py, data/pix2pix_dataset.py, data/{ade20k,celebahq,deepfashion}_dataset.py):
the draws from `random` happen in the same order (crop x, crop y, flip per label map; one reference draw per item;
the DeepFashion reference lists draw while they are read), and the resampling goes through the same PIL filters
(BICUBIC for photographs, NEAREST for label maps, BILINEAR for the pose distance maps).

The reference lists are read from ./data/<mode>_ref{,_test}.txt relative to the working directory, where the
reference keeps them, so its list files drop in unchanged.
"""
import math
import os
import random
import re

import numpy as np
import torch
import torch.utils.data
import torchvision.transforms.functional as TF
from PIL import Image

IMG_EXTENSIONS = (".jpg", ".JPG", ".jpeg", ".JPEG", ".png", ".PNG", ".ppm", ".PPM", ".bmp", ".BMP", ".tiff", ".webp")


def natural_sort(items):
    """In place, digit runs compared as numbers ("img2" < "img10")."""
    items.sort(key=lambda s: [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", s)])


def list_images(root, read_cache=False):
    """Every image file under root, walking directories in sorted order.  With read_cache, a root/files.list (one path
    per line) is taken verbatim instead of walking."""
    if read_cache:
        cached = os.path.join(root, "files.list")
        if os.path.isfile(cached):
            with open(cached) as f:
                return f.read().splitlines()
    assert os.path.isdir(root), "%s is not a valid directory" % root
    found = []
    for folder, _, files in sorted(os.walk(root, followlinks=True)):
        found += [os.path.join(folder, f) for f in files if f.endswith(IMG_EXTENSIONS)]
    return found


# ---------------------------------------------------------------------------------------------------------------------
# shared transforms

def get_params(opt, size):
    """Crop position and flip for an image of PIL size (w, h).  Draws randint, randint, random -- always, also when the
    crop is empty or flipping is off, so the stream of draws does not depend on the options."""
    w, h = size
    new_w, new_h = w, h
    if opt.preprocess_mode == "resize_and_crop":
        new_w = new_h = opt.load_size
    elif opt.preprocess_mode == "scale_width_and_crop":
        new_w, new_h = opt.load_size, opt.load_size * h // w
    elif opt.preprocess_mode == "scale_shortside_and_crop":
        short, long_ = min(w, h), max(w, h)
        long_ = int(opt.load_size * long_ / short)
        new_w, new_h = (short, long_) if w == short else (long_, short)
    x = random.randint(0, max(0, new_w - opt.crop_size))
    y = random.randint(0, max(0, new_h - opt.crop_size))
    return {"crop_pos": (x, y), "flip": random.random() > 0.5}


def _resize_geometry(opt, img, method):
    mode = opt.preprocess_mode
    w, h = img.size
    if "resize" in mode:
        img = img.resize((opt.load_size, opt.load_size), method)
    elif "scale_width" in mode:
        if w != opt.load_size:
            img = img.resize((opt.load_size, int(opt.load_size * h / w)), method)
    elif "scale_shortside" in mode:
        short, long_ = min(w, h), max(w, h)
        if short != opt.load_size:
            long_ = int(opt.load_size * long_ / short)
            img = img.resize((short, long_) if w == short else (long_, short), method)
    return img


def transform(opt, params, img, method=Image.BICUBIC, normalize=True):
    """PIL image -> float tensor: resize / crop per --preprocess_mode, the flip (training only), ToTensor and, for
    photographs, Normalize(0.5, 0.5) to [-1, 1]."""
    img = _resize_geometry(opt, img, method)
    if "crop" in opt.preprocess_mode:
        x, y = params["crop_pos"]
        img = img.crop((x, y, x + opt.crop_size, y + opt.crop_size))
    if opt.preprocess_mode == "none":  # round both sides to a multiple of 32
        w, h = img.size
        nw, nh = int(round(w / 32) * 32), int(round(h / 32) * 32)
        if (nw, nh) != (w, h):
            img = img.resize((nw, nh), method)
    if opt.preprocess_mode == "fixed":
        img = img.resize((opt.crop_size, round(opt.crop_size / opt.aspect_ratio)), method)
    if opt.isTrain and not opt.no_flip and params["flip"]:
        img = img.transpose(Image.FLIP_LEFT_RIGHT)
    t = TF.to_tensor(img)
    if normalize:
        t = TF.normalize(t, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5))
    return t


def _read_list(path):
    with open(path) as f:
        return f.readlines()


# ---------------------------------------------------------------------------------------------------------------------
# pairing

class PairedDataset(torch.utils.data.Dataset):
    """Label map + photograph per item, with an exemplar: with probability real_reference_probability (always at test)
    one from the reference list -- the hard one below hard_reference_probability, else the easy one -- otherwise the
    item itself (self_ref = 1)."""
    natural_order = True
    train_test_folder = ("", "")

    def __init__(self, opt):
        self.opt = opt
        labels, images = self.get_paths(opt)
        if self.natural_order:
            natural_sort(labels)
            natural_sort(images)
        labels, images = labels[:opt.max_dataset_size], images[:opt.max_dataset_size]
        if not opt.no_pairing_check:
            for a, b in zip(labels, images):
                assert self.paths_match(a, b), \
                    "label %s and image %s do not look like a pair (use --no_pairing_check to skip this check)" % (a, b)
        self.label_paths, self.image_paths = labels, images
        test = opt.phase == "test"
        self.real_reference_probability = 1 if test else opt.real_reference_probability
        self.hard_reference_probability = 0 if test else opt.hard_reference_probability
        self.ref_dict = self.get_ref(opt)

    @staticmethod
    def paths_match(a, b):
        return os.path.splitext(os.path.basename(a))[0] == os.path.splitext(os.path.basename(b))[0]

    def __len__(self):
        return len(self.label_paths)

    def ref_key(self, image_path):
        return os.path.basename(image_path)

    def ref_image_path(self, image_path, name):
        old, new = self.train_test_folder[1], self.train_test_folder[0]
        return os.path.dirname(image_path).replace(old, new) + "/" + name

    def ref_label_path(self, ref_path):
        return self.imgpath_to_labelpath(ref_path.replace(".jpg", ".png"))

    def imgpath_to_labelpath(self, path):
        return path

    def get_label_tensor(self, path):
        label = Image.open(path)
        params = get_params(self.opt, label.size)
        t = transform(self.opt, params, label, method=Image.NEAREST, normalize=False) * 255.0
        t[t == 255] = self.opt.label_nc  # 'unknown' becomes label_nc
        return t, params

    def _exemplar(self, path):
        """(exemplar tensor, its label map) for the photograph at path."""
        image = Image.open(path).convert("RGB")
        label, params = self.get_label_tensor(self.ref_label_path(path))
        return transform(self.opt, params, image), label

    def self_pair(self, image_path):
        """--video_like only (DeepFashion): another frame of the same clip, or None."""
        return None

    def __getitem__(self, index):
        label_path, image_path = self.label_paths[index], self.image_paths[index]
        label, params = self.get_label_tensor(label_path)
        if not self.opt.no_pairing_check:
            assert self.paths_match(label_path, image_path), (label_path, image_path)
        image = Image.open(image_path).convert("RGB")
        image_tensor = transform(self.opt, params, image)

        p = random.random()
        if p < self.real_reference_probability or self.opt.phase == "test":
            refs = self.ref_dict[self.ref_key(image_path)]
            name = refs[1] if p < self.hard_reference_probability else refs[0]  # hard, else easy
            ref, label_ref = self._exemplar(self.ref_image_path(image_path, name))
            self_ref = torch.zeros_like(ref)
        else:
            pair = self.self_pair(image_path)
            if pair is not None:
                ref, label_ref = self._exemplar(pair)
            else:
                label_ref, params = self.get_label_tensor(label_path)
                ref = transform(self.opt, params, image)
            self_ref = torch.ones_like(ref)
        return {"label": label, "image": image_tensor, "path": image_path, "self_ref": self_ref, "ref": ref,
                "label_ref": label_ref}


def _ref_lines(mode, opt):
    return _read_list("./data/%s_ref%s.txt" % (mode, "_test" if opt.phase == "test" else ""))


def _easy_hard_refs(lines, opt):
    """key -> [easy, hard] (training) or every listed reference (test)."""
    out = {}
    for line in lines:
        items = line.strip().split(",")
        out[items[0]] = items[1:] if opt.phase == "test" else [items[1], items[-1]]
    return out


class ADE20KDataset(PairedDataset):
    """<dataroot>/{training,validation}/ADE_{train,val}_*.{jpg,png}; label value 255 becomes the don't-care class
    label_nc."""
    train_test_folder = ("training", "validation")

    def get_paths(self, opt):
        test = opt.phase == "test"
        tag = "_%s_" % ("val" if test else "train")
        found = sorted(list_images(opt.dataroot + "/" + ("validation" if test else "training"), read_cache=not test))
        found = [p for p in found if tag in p]
        return [p for p in found if p.endswith(".png")], [p for p in found if p.endswith(".jpg")]

    def get_ref(self, opt):
        return _easy_hard_refs(_ref_lines("ade20k", opt), opt)


class CelebAHQDataset(PairedDataset):
    """<dataroot>/{train,val}.txt lists image ids; photographs in CelebA-HQ-img/<id>.jpg, class ids in
    CelebAMask-HQ-mask-anno/all_parts_except_glasses/<id:05d>.png and the glasses mask, where there is one, in
    CelebAMask-HQ-mask-anno/<id // 2000>/<id:05d>_eye_g.png.  The label is the 2-channel [ids, glasses] map."""
    natural_order = False

    def get_paths(self, opt):
        ids = [s.strip() for s in _read_list(os.path.join(opt.dataroot, "train.txt" if opt.phase == "train"
                                                          else "val.txt"))]
        return ([os.path.join(opt.dataroot, "CelebAMask-HQ-mask-anno", "all_parts_except_glasses", i.zfill(5) + ".png")
                 for i in ids],
                [os.path.join(opt.dataroot, "CelebA-HQ-img", i + ".jpg") for i in ids])

    def get_ref(self, opt):
        return _easy_hard_refs(_ref_lines("celebahq", opt), opt)

    def get_label_tensor(self, path):
        ids = Image.open(path).convert("L")
        root, name = path.replace("\\", "/").split("all_parts_except_glasses/")
        idx = name.split(".")[0]
        glasses_path = os.path.join(root, str(int(idx) // 2000), idx + "_eye_g.png")
        if os.path.exists(glasses_path):
            glasses = Image.open(glasses_path).convert("L")
        else:
            glasses = Image.fromarray(np.zeros(ids.size, dtype=np.uint8))
        params = get_params(self.opt, ids.size)
        ids_t = transform(self.opt, params, ids, method=Image.NEAREST, normalize=False) * 255.0
        glasses_t = transform(self.opt, params, glasses, method=Image.NEAREST, normalize=False)
        return torch.cat((ids_t, glasses_t), dim=0), params

    def imgpath_to_labelpath(self, path):
        root, name = path.split("CelebA-HQ-img/")
        return os.path.join(root, "CelebAMask-HQ-mask-anno", "all_parts_except_glasses",
                            name.split(".")[0].zfill(5) + ".png")


# OpenPose's 18 keypoints: the joint pairs (1-based) of the 17 limbs that are drawn, and one BGR colour per keypoint
# (limb i is drawn in the colour of keypoint i)
_LIMBS = [[2, 3], [2, 6], [3, 4], [4, 5], [6, 7], [7, 8], [2, 9], [9, 10], [10, 11], [2, 12], [12, 13], [13, 14],
          [2, 1], [1, 15], [15, 17], [1, 16], [16, 18]]
_COLORS = [[255, 0, 0], [255, 85, 0], [255, 170, 0], [255, 255, 0], [170, 255, 0], [85, 255, 0], [0, 255, 0],
           [0, 255, 85], [0, 255, 170], [0, 255, 255], [0, 170, 255], [0, 85, 255], [0, 0, 255], [85, 0, 255],
           [170, 0, 255], [255, 0, 255], [255, 0, 170], [255, 0, 85]]
_LIMB_HALF_WIDTH = 4  # pixels; also the radius of a keypoint's disc


def _limb_polygon(cv2, p, q):
    """The limb from keypoint p to keypoint q ((x, y) each, float64) as a closed polygon: an ellipse whose long axis
    joins them, with integer centre, semi-axes and angle in degrees as cv2.ellipse2Poly takes them."""
    dx, dy = p[0] - q[0], p[1] - q[1]
    centre = (int(np.mean([p[0], q[0]])), int(np.mean([p[1], q[1]])))
    semi_axes = (int((dy ** 2 + dx ** 2) ** 0.5 / 2), _LIMB_HALF_WIDTH)
    return cv2.ellipse2Poly(centre, semi_axes, int(math.degrees(math.atan2(dy, dx))), 0, 360, 1)


def render_pose(candidate, subset, shape):
    """The stick figure of one OpenPose detection on a black BGR image of `shape`, and one uint8 mask per limb.

    candidate: rows (x, y, ...) of detected keypoints; subset: for each of the 18 keypoints its row in candidate, or
    -1 when it was not detected.  Keypoints are discs.  Each limb is blended over the figure so far at 60 % opacity;
    a limb with an undetected end is skipped and its mask is empty.  Each mask holds 255 inside the limb's polygon,
    after the same 0.4 / 0.6 cv2.addWeighted pass (of the mask with itself) as the figure."""
    import cv2
    figure = np.zeros(shape, np.uint8)
    for k, row in enumerate(subset[:18].astype(int)):
        if row != -1:
            x, y = candidate[row][0:2]
            cv2.circle(figure, (int(x), int(y)), _LIMB_HALF_WIDTH, _COLORS[k], thickness=-1)
    masks = []
    for k, ends in enumerate(_LIMBS):
        rows = subset[np.array(ends) - 1]
        mask = np.zeros(shape[:2], np.uint8)
        if -1 not in rows:
            p, q = candidate[rows.astype(int)]
            polygon = _limb_polygon(cv2, p, q)
            limb = figure.copy()
            cv2.fillConvexPoly(limb, polygon, _COLORS[k])
            figure = cv2.addWeighted(figure, 0.4, limb, 0.6, 0)
            cv2.fillConvexPoly(mask, polygon, 255)
            mask = cv2.addWeighted(mask, 0.4, mask, 0.6, 0)
        masks.append(mask)
    return figure, masks


class DeepFashionDataset(PairedDataset):
    """<dataroot>/{train,val}.txt lists img/<...>.jpg paths (backslashes allowed); the pose of each is in
    pose/<...>_{candidate,subset}.txt.  The label is 20 float channels: the stick figure (RGB) and one distance map per
    limb.  With --video_like a self-reference is another frame of the same clip (./data/deepfashion_self_pair.txt)."""
    natural_order = False

    def get_paths(self, opt):
        lines = _read_list(os.path.join(opt.dataroot, "train.txt" if opt.phase == "train" else "val.txt"))
        images, labels = [], []
        for line in lines:
            s = line.strip()
            images.append(os.path.join(opt.dataroot, s.replace("\\", "/")))
            labels.append(os.path.join(opt.dataroot,
                                       s.replace("img", "pose").replace(".jpg", "_{}.txt").replace("\\", "/")))
        return labels, images

    def ref_key(self, image_path):
        return image_path.replace("\\", "/").split("DeepFashion/")[-1]

    def ref_image_path(self, image_path, name):
        return os.path.join(self.opt.dataroot, name)

    def ref_label_path(self, ref_path):
        return self.imgpath_to_labelpath(ref_path)

    def _sample_names(self):
        return [p.split("DeepFashion/")[-1] for p in random.sample(self.image_paths, min(len(self.image_paths), 20))]

    def get_ref(self, opt):
        test = opt.phase == "test"
        lines = [s.strip() for s in _ref_lines("deepfashion", opt)]
        ref = {}
        if opt.video_like:
            with open("./data/deepfashion_self_pair.txt") as f:
                pairs = {}
                for s in f.readlines():
                    items = s.strip().split(",")
                    pairs[items[0]] = items[1:]
            for line in lines:
                items = line.split(",")
                first = [t.replace("\\", "/") for t in pairs[items[0]]] if items[0] in pairs \
                    else [items[-1].replace("\\", "/")]
                ref[items[0].replace("\\", "/")] = first + self._sample_names()
        else:
            for line in lines:
                items = line.split(",")
                if test:
                    val = [t.replace("\\", "/") for t in items[1:]]
                else:
                    val = [items[-1].replace("\\", "/"),
                           random.choice(self.image_paths).split("DeepFashion/")[-1].replace("\\", "/")]
                ref[items[0].replace("\\", "/")] = val
        return ref

    def self_pair(self, image_path):
        if not self.opt.video_like:
            return None
        key = self.ref_key(image_path)
        name = self.ref_dict[key][0]
        if os.path.dirname(name) == os.path.dirname(key) and \
                os.path.basename(name).split("_")[0] == os.path.basename(key).split("_")[0]:
            return os.path.join(self.opt.dataroot, name)
        return None

    def get_label_tensor(self, path):
        """[stick figure (RGB), 17 limb distance maps] at load_size, cropped and flipped together.  A distance map
        holds the L1 (3x3 chamfer) distance to the limb, divided by 3 and clipped to 255."""
        import cv2
        shape = cv2.imread(self.labelpath_to_imgpath(path)).shape
        figure, masks = render_pose(np.loadtxt(path.format("candidate")), np.loadtxt(path.format("subset")), shape)
        pose = Image.fromarray(cv2.cvtColor(figure, cv2.COLOR_BGR2RGB)).resize((self.opt.load_size,) * 2,
                                                                                resample=Image.NEAREST)
        params = get_params(self.opt, pose.size)
        dists = []
        for mask in masks:
            d = np.clip(cv2.distanceTransform(255 - mask, cv2.DIST_L1, 3) / 3, 0, 255).astype(np.uint8)
            dists.append(transform(self.opt, params, Image.fromarray(d), method=Image.BILINEAR, normalize=False))
        pose_t = transform(self.opt, params, pose, method=Image.NEAREST, normalize=False)
        return torch.cat([pose_t] + dists, dim=0), params

    def imgpath_to_labelpath(self, path):
        return path.replace("\\", "/").replace("/img/", "/pose/").replace(".jpg", "_{}.txt")

    def labelpath_to_imgpath(self, path):
        return path.replace("\\", "/").replace("/pose/", "/img/").replace("_{}.txt", ".jpg")


READERS = {"ade20k": ADE20KDataset, "celebahq": CelebAHQDataset, "deepfashion": DeepFashionDataset}
