# -*- coding: utf-8 -*-
"""Region samplers of the reference (lfd/data_pipeline/sampler/region_sampler.py), split in two.

`draw(sample)` makes every random draw and all the integer box arithmetic of the reference, in its order, without touching pixels,
and returns a `RegionDraw`: the resize scale s, the crop window in resized coordinates, the boxes and labels that survive the crop
and the meta keys the sampler adds.  The data loader turns a draw into pixels on the GPU (lfd_input_batch).
`__call__(sample)` keeps the reference's host contract: numpy image in, cv2.resize + crop_from_image, numpy image out.
"""
import collections
import math
import random

import numpy

__all__ = ['BaseRegionSampler',
           'TypicalCOCOTrainingRegionSampler',
           'RandomBBoxCropRegionSampler',
           'RandomBBoxCropWithRangeSelectionRegionSampler',
           'IdleRegionSampler',
           'RegionDraw',
           'resize_plan',
           'crop_from_image']

# scale: the factor of cv2.resize(fx = fy = scale); crop: (x, y, w, h) in resized coordinates, w x h is the output size;
# bboxes / bbox_labels: what the sample holds afterwards (None: the key is absent); meta: keys the sampler adds to the sample
RegionDraw = collections.namedtuple('RegionDraw', ['scale', 'crop', 'bboxes', 'bbox_labels', 'meta'])

RESIZE_COPY, RESIZE_LINEAR, RESIZE_AREA2 = 0, 1, 2


def resize_plan(height, width, scale):
    """(mode, resized height, resized width) of cv2.resize(image, (0, 0), fx=scale, fy=scale) on uint8: cv2 rounds the size half to
    even, copies when it is unchanged and switches INTER_LINEAR to INTER_AREA when 1 / scale is exactly 2."""
    dw, dh = int(round(width * scale)), int(round(height * scale))
    if dw <= 0 or dh <= 0:
        raise ValueError('resize scale %r makes a %dx%d image empty' % (scale, height, width))
    if dw == width and dh == height:
        return RESIZE_COPY, dh, dw
    inv = 1.0 / scale
    if abs(inv - round(inv)) < numpy.finfo(numpy.float64).eps and round(inv) == 2:
        return RESIZE_AREA2, dh, dw
    return RESIZE_LINEAR, dh, dw


def crop_from_image(image, crop_region):
    """The (x, y, w, h) region of `image`; the parts outside the image are zero."""
    im_h, im_w = image.shape[:2]
    x, y, w, h = crop_region
    out = numpy.zeros((h, w) + image.shape[2:], dtype=image.dtype)
    out[max(0, -y):min(h, im_h - y), max(0, -x):min(w, im_w - x)] = image[max(0, y):min(im_h, h + y), max(0, x):min(im_w, w + x)]
    return out


def _shape(sample, image_shape):
    return tuple(image_shape[:2]) if image_shape is not None else tuple(sample['image'].shape[:2])


def _crop_boxes(scaled, labels, crop_x, crop_y, crop_size):
    """Boxes clipped to the crop, minus one pixel on the far sides; boxes left with w or h <= 1 are dropped."""
    boxes, kept = [], []
    for i, (bx, by, bw, bh) in enumerate(scaled):
        nx, ny = max(0, bx - crop_x), max(0, by - crop_y)
        nw = min(crop_size, bx + bw - crop_x) - nx - 1
        nh = min(crop_size, by + bh - crop_y) - ny - 1
        if nw <= 1 or nx >= crop_size or nh <= 1 or ny >= crop_size:
            continue
        boxes.append([nx, ny, nw, nh])
        kept.append(labels[i])
    return (boxes, kept) if boxes else (None, None)


def _scale_boxes(bboxes, s):
    return [[int(b[0] * s), int(b[1] * s), math.ceil(b[2] * s), math.ceil(b[3] * s)] for b in bboxes]


def _crop_around(target, crop_size):
    w_range, h_range = crop_size - target[2], crop_size - target[3]
    crop_x = target[0] - random.randint(min(0, w_range), max(0, w_range))
    crop_y = target[1] - random.randint(min(0, h_range), max(0, h_range))
    return crop_x, crop_y


class BaseRegionSampler(object):
    def draw(self, sample, image_shape=None):
        """-> RegionDraw; image_shape (h, w) stands in for sample['image'].shape when the image is not decoded."""
        raise NotImplementedError

    def __call__(self, sample):
        """Host path, numpy in and out: replaces sample['image'] by its region, updates boxes, labels and meta keys."""
        import cv2
        d = self.draw(sample)
        if not isinstance(self, IdleRegionSampler):
            sample['image'] = crop_from_image(cv2.resize(sample['image'], (0, 0), fx=d.scale, fy=d.scale), d.crop)
        return apply_draw(sample, d)


def apply_draw(sample, d):
    """The non-pixel part of a region sampler's result: boxes, labels and meta keys."""
    if d.bboxes is not None:
        sample['bboxes'], sample['bbox_labels'] = d.bboxes, d.bbox_labels
    elif 'bboxes' in sample:
        del sample['bboxes'], sample['bbox_labels']
    sample.update(d.meta)
    return sample


class TypicalCOCOTrainingRegionSampler(BaseRegionSampler):
    """Resize keeping the aspect ratio so that the shorter edge becomes a random length in resize_shorter_range, unless the longer
    edge would exceed resize_longer_limit; the output is padded to a multiple of pad_divisor."""

    def __init__(self, resize_shorter_range=(800,), resize_longer_limit=1333, pad_divisor=32):
        assert isinstance(resize_shorter_range, tuple)
        assert max(resize_shorter_range) <= resize_longer_limit
        assert pad_divisor > 0
        self._pad_divisor = pad_divisor
        self._resize_shorter_min = min(resize_shorter_range)
        self._resize_shorter_max = max(resize_shorter_range)
        self._resize_longer_limit = resize_longer_limit

    def draw(self, sample, image_shape=None):
        h, w = _shape(sample, image_shape)
        shorter_target = random.randint(self._resize_shorter_min, self._resize_shorter_max)
        s = min(self._resize_longer_limit / max(h, w), shorter_target / min(h, w))
        _, dh, dw = resize_plan(h, w, s)
        boxes = None
        if 'bboxes' in sample:
            boxes = [[int(b[0] * s), int(b[1] * s), max(int(b[2] * s), 1), max(int(b[3] * s), 1)] for b in sample['bboxes']]
        crop = (0, 0, math.ceil(dw / self._pad_divisor) * self._pad_divisor, math.ceil(dh / self._pad_divisor) * self._pad_divisor)
        meta = dict(resize_scale=s, resized_height=int(h * s), resized_width=int(w * s))
        return RegionDraw(s, crop, boxes, sample.get('bbox_labels') if boxes is not None else None, meta)


class RandomBBoxCropRegionSampler(BaseRegionSampler):
    """With probability resize_prob resize by a uniform scale in resize_range, then crop crop_size x crop_size around a random box
    (anywhere for a sample without boxes)."""

    def __init__(self, crop_size, resize_range=(0.5, 1.5), resize_prob=1.0):
        assert isinstance(crop_size, int)
        assert isinstance(resize_range, (tuple, list))
        assert 0 <= resize_prob <= 1.
        self._crop_size = crop_size
        self._resize_range = resize_range
        self._resize_prob = resize_prob

    def draw(self, sample, image_shape=None):
        h, w = _shape(sample, image_shape)
        if random.random() < self._resize_prob:
            s = random.random() * (self._resize_range[1] - self._resize_range[0]) + self._resize_range[0]
        else:
            s = 1.0
        _, dh, dw = resize_plan(h, w, s)
        scaled = _scale_boxes(sample.get('bboxes', []), s)
        target = random.choice(scaled) if scaled else [0, 0, dw, dh]
        crop_x, crop_y = _crop_around(target, self._crop_size)
        boxes, labels = _crop_boxes(scaled, sample.get('bbox_labels', []), crop_x, crop_y, self._crop_size)
        return RegionDraw(s, (crop_x, crop_y, self._crop_size, self._crop_size), boxes, labels, {})


class RandomBBoxCropWithRangeSelectionRegionSampler(BaseRegionSampler):
    """Pick a random box, resize so that its side (range_mode) falls in a randomly selected detection range, then crop
    crop_size x crop_size around it; samples without boxes resize by a uniform scale in neg_resize_range."""

    def __init__(self, crop_size, detection_ranges, range_mode='longer', neg_resize_range=(0.5, 3), range_selection_probs=None, lock_threshold=None):
        assert isinstance(crop_size, int)
        assert isinstance(detection_ranges, (tuple, list))
        assert range_mode in ['shorter', 'longer', 'sqrt']
        assert isinstance(neg_resize_range, (tuple, list)) and len(neg_resize_range) == 2
        if range_selection_probs is not None:
            assert len(detection_ranges) == len(range_selection_probs)
        if lock_threshold is not None:
            assert isinstance(lock_threshold, int)
        self._crop_size = crop_size
        self._detection_ranges = detection_ranges
        self._range_mode = range_mode
        self._range_lower_bound = detection_ranges[0][0]
        self._range_upper_bound = detection_ranges[-1][1]
        if range_selection_probs is None:
            self._range_selection_probs = [1. / len(detection_ranges)] * len(detection_ranges)
        else:
            self._range_selection_probs = [p / sum(range_selection_probs) for p in range_selection_probs]
        self._neg_resize_range = neg_resize_range
        self._lock_threshold = lock_threshold

    def _scale_for(self, box):
        side = {'shorter': lambda: min(box[-2:]), 'longer': lambda: max(box[-2:]), 'sqrt': lambda: (box[-2] * box[-1]) ** 0.5}[self._range_mode]()
        if side <= self._range_lower_bound:
            return 1.0
        if self._lock_threshold and side <= self._lock_threshold:
            return random.randint(self._range_lower_bound, side) / side
        if side >= self._range_upper_bound and random.random() > 0.9:
            return (self._range_upper_bound + random.randint(0, self._range_upper_bound * 0.5)) / side
        target_range = random.choices(self._detection_ranges, self._range_selection_probs)[0]
        return random.randint(target_range[0], target_range[1]) / side

    def draw(self, sample, image_shape=None):
        h, w = _shape(sample, image_shape)
        bboxes = sample.get('bboxes', [])
        target_index = -1
        if bboxes:
            target_index = random.randint(0, len(bboxes) - 1)
            s = self._scale_for(bboxes[target_index])
        else:
            s = random.random() * (self._neg_resize_range[1] - self._neg_resize_range[0]) + self._neg_resize_range[0]
        _, dh, dw = resize_plan(h, w, s)
        scaled = _scale_boxes(bboxes, s)
        target = scaled[target_index] if scaled else [0, 0, dw, dh]
        crop_x, crop_y = _crop_around(target, self._crop_size)
        boxes, labels = _crop_boxes(scaled, sample.get('bbox_labels', []), crop_x, crop_y, self._crop_size)
        return RegionDraw(s, (crop_x, crop_y, self._crop_size, self._crop_size), boxes, labels, {})


class IdleRegionSampler(BaseRegionSampler):
    """The whole image, unchanged (evaluation)."""

    def draw(self, sample, image_shape=None):
        h, w = _shape(sample, image_shape)
        return RegionDraw(1.0, (0, 0, w, h), sample.get('bboxes'), sample.get('bbox_labels'),
                          dict(resize_scale=1., resized_height=h, resized_width=w))
