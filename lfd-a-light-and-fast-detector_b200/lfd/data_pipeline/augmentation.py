# -*- coding: utf-8 -*-
import collections
import random

import numpy

__all__ = ['simple_normalize_pipeline']


def simple_normalize_pipeline(sample):
    """(x/255 - 0.5)/0.5 on the BGR uint8 image -> float32 HWC
    (lfd/data_pipeline/augmentation/augmentation_pipeline.py:31-36, albumentations.Normalize(mean=.5, std=.5))."""
    img = sample['image'].astype(numpy.float32)
    sample['image'] = (img - numpy.float32(127.5)) * numpy.float32(1.0 / 127.5)
    return sample


# ------------------------------------------------------------------------------------------------------------------------------
# Declarative stand-ins for the albumentations transforms the reference's pipelines use (augmentation_pipeline.py,
# new_augmentations.py).  The data loader reads them (flip probability, channel order, mean, std, max_pixel) and runs them inside
# the input kernel; called on a host sample they apply the same operation with numpy.  albumentations' own consumption of the
# random stream (Compose and every transform draw for their `p`) is not reproduced: only HorizontalFlip draws, random.random() < p.

__all__ += ['Compose', 'HorizontalFlip', 'Normalize', 'BboxParams', 'BGR2RGB',
            'typical_coco_train_pipeline', 'typical_coco_val_pipeline', 'simple_widerface_train_pipeline',
            'simple_widerface_val_pipeline', 'caffe_imagenet_normalize', 'standard_normalize', 'simple_normalize', 'bbox_param']


class BboxParams(object):
    def __init__(self, format='coco', label_fields=None, **kwargs):
        assert format == 'coco', 'only coco boxes (x, y, w, h) are supported'
        self.format, self.label_fields = format, label_fields


class HorizontalFlip(object):
    def __init__(self, always_apply=False, p=0.5):
        self.p = 1.0 if always_apply else p

    def apply(self, sample, flip):
        if flip:
            w = sample['image'].shape[1]
            sample['image'] = numpy.ascontiguousarray(sample['image'][:, ::-1])
            if 'bboxes' in sample:
                sample['bboxes'] = [(w - b[0] - b[2], b[1], b[2], b[3]) for b in sample['bboxes']]
        return sample


class BGR2RGB(object):
    def __init__(self, always_apply=False, p=1.):
        self.p = 1.0 if always_apply else p

    def apply(self, sample):
        sample['image'] = numpy.ascontiguousarray(sample['image'][..., ::-1])
        return sample


class Normalize(object):
    def __init__(self, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), max_pixel_value=255.0, always_apply=False, p=1.0):
        self.mean, self.std, self.max_pixel_value, self.p = mean, std, max_pixel_value, 1.0 if always_apply else p

    def constants(self):
        """(mean * max_pixel, reciprocal(std * max_pixel)) in float32, as albumentations.normalize computes them."""
        m = numpy.array(self.mean, numpy.float32) * numpy.float32(self.max_pixel_value)
        d = numpy.reciprocal(numpy.array(self.std, numpy.float32) * numpy.float32(self.max_pixel_value), dtype=numpy.float32)
        return m, d

    def apply(self, sample):
        m, d = self.constants()
        sample['image'] = (sample['image'].astype(numpy.float32) - m) * d
        return sample


class _Probe(object):
    """Stands in for the image when the data loader asks a pipeline which Compose it would run (see Compose.__call__)."""


class Compose(object):
    def __init__(self, transforms, bbox_params=None, p=1.0):
        self.transforms, self.bbox_params, self.p = list(transforms), bbox_params, p

    def __call__(self, sample=None, **kwargs):
        sample = dict(sample if sample is not None else kwargs)
        if isinstance(sample.get('image'), _Probe):
            return {'image': self}
        for t in self.transforms:
            if isinstance(t, HorizontalFlip):
                t.apply(sample, random.random() < t.p)
            else:
                t.apply(sample)
        return sample

    def device_spec(self):
        """(flip_p or None, swap_rb, mean[3], scale[3]) when the input kernel can run this pipeline, else None: at most one flip,
        BGR2RGB and Normalize with p = 1, Normalize (at most one) last."""
        flip_p, swap, norm = None, False, None
        for i, t in enumerate(self.transforms):
            if isinstance(t, HorizontalFlip) and flip_p is None:
                flip_p = t.p
            elif isinstance(t, BGR2RGB) and t.p == 1:
                swap = not swap
            elif isinstance(t, Normalize) and t.p == 1 and i == len(self.transforms) - 1:
                norm = t
            else:
                return None
        mean, scale = norm.constants() if norm is not None else (numpy.zeros(3, numpy.float32), numpy.ones(3, numpy.float32))
        return flip_p, swap, mean, scale


def pipeline_device_spec(pipeline, with_bboxes):
    """What the input kernel needs to run `pipeline` on a sample with / without boxes, or None when it has to run on the host:
    the pipeline is None, a Compose of the stand-ins above, or a function that only picks such a Compose from the sample's keys."""
    if pipeline is None:
        return None, False, numpy.zeros(3, numpy.float32), numpy.ones(3, numpy.float32)
    compose = pipeline
    if not isinstance(pipeline, Compose):
        probe = {'image': _Probe()}
        if with_bboxes:
            probe.update(bboxes=[], bbox_labels=[])
        try:
            compose = pipeline(probe)['image']
        except Exception:
            return None
    return compose.device_spec() if isinstance(compose, Compose) else None


# What the stem kernels can do to a uint8 BGR frame while they read it: network input channel c of a pixel =
# (float32(byte[2 - c if swap_rb else c]) - mean[c]) * scale[c], i.e. BGR2RGB.apply (optional) then Normalize.apply.  mean / scale: 3-tuples
# of floats holding float32 values (Normalize.constants()); hashable, so a transform can be part of a plan's cache key.
InputTransform = collections.namedtuple('InputTransform', 'swap_rb mean scale')
__all__ += ['InputTransform', 'input_transform_of']


def _gray_transform(swap, mean, scale):
    """The transform of a gray (1-channel) model: (byte - mean) * scale with no channel swap, kept as three equal constants, which is what
    the library takes for a 1-channel image (include/lfd_b200.h).  BGR2RGB, or unequal per-channel constants, have no meaning on one channel."""
    mean, scale = tuple(float(v) for v in numpy.atleast_1d(mean)), tuple(float(v) for v in numpy.atleast_1d(scale))
    if swap:
        raise ValueError('a gray (1-channel) model has no channel order: BGR2RGB cannot run on its input')
    if len(set(mean)) != 1 or len(set(scale)) != 1:
        raise ValueError('a gray (1-channel) model takes a Normalize with one constant or three equal ones (got mean %r, scale %r)' % (mean, scale))
    return InputTransform(False, (mean[0],) * 3, (scale[0],) * 3)


def input_transform_of(pipeline, allow_flip=False, channels=3):
    """pipeline -> the InputTransform the stem kernels run in its place; None -> None (the kernels' default, simple_normalize); an
    InputTransform is returned as it is.  Raises ValueError for a pipeline Compose.device_spec() cannot express, and for one with a
    HorizontalFlip unless allow_flip (the training loader, whose input kernel does the flip before the stem sees the batch).
    channels=1: the transform of a gray model's one channel -- a final Normalize with one constant or three equal ones, no BGR2RGB
    (ValueError otherwise)."""
    if pipeline is None:
        return None
    if isinstance(pipeline, InputTransform):
        return pipeline if channels == 3 else _gray_transform(pipeline.swap_rb, pipeline.mean, pipeline.scale)
    spec = pipeline_device_spec(pipeline, False)
    if spec is None:
        raise ValueError('the stem kernels cannot run this pipeline on uint8 frames: it must be a Compose (or a function that picks one by the '
                         "sample's keys) of BGR2RGB and one final Normalize, each with p = 1 (got %r)" % (pipeline,))
    flip_p, swap, mean, scale = spec
    if flip_p is not None and not allow_flip:
        raise ValueError('the stem kernels cannot run a HorizontalFlip (p = %g): the input transform is a channel swap and a normalisation' % flip_p)
    if channels == 1:
        return _gray_transform(swap, mean, scale)
    return InputTransform(bool(swap), tuple(float(v) for v in mean), tuple(float(v) for v in scale))


random_horizon_flip = HorizontalFlip(p=0.5)
caffe_imagenet_normalize = Normalize(mean=(102.9801, 115.9465, 122.7717), std=(1.0, 1.0, 1.0), max_pixel_value=1.0, p=1.0)
standard_normalize = Normalize(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), max_pixel_value=255.0, p=1.0)
simple_normalize = Normalize(mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), max_pixel_value=255.0, p=1.0)
bbox_param = BboxParams(format='coco', label_fields=['bbox_labels'])

# the reference picks a Compose with or without bbox_params by the sample's keys; the stand-in handles both with one
typical_coco_train_pipeline = Compose([random_horizon_flip, caffe_imagenet_normalize], bbox_params=bbox_param, p=1.)
typical_coco_val_pipeline = Compose([caffe_imagenet_normalize], bbox_params=bbox_param, p=1.)
simple_widerface_train_pipeline = Compose([random_horizon_flip, simple_normalize], bbox_params=bbox_param, p=1.)
simple_widerface_val_pipeline = Compose([simple_normalize], bbox_params=bbox_param, p=1.)
