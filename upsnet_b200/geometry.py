"""Per-image geometry of the reference's loader: the scale rule of prep_im_for_blob and, for the test phase, everything
that follows from one original image size -- the resized and padded network input, im_info, the size the label maps are
restored to and the size im_post pastes the masks at.  Host arithmetic only; the training loader (TrainingSample) and
the mixed-size PipelinedEngine share it."""
from collections import namedtuple

import numpy as np

ImageGeometry = namedtuple("ImageGeometry", "scale resized padded im_info restored im_post")


def prep_scale(target_size, max_size, h, w):
    """prep_im_for_blob's scale of an h x w image for one target size (dataset/base_dataset.py:158-168): float64
    target / min(h, w), replaced by max_size / max(h, w) when np.round(scale * max(h, w)) > max_size."""
    size_min, size_max = min(h, w), max(h, w)
    s = float(target_size) / float(size_min)
    if np.round(s * size_max) > max_size:
        s = float(max_size) / float(size_max)
    return s


def image_geometry(h, w, target_size, max_size, stride=32):
    """The test-phase geometry of one h x w image:
      scale     prep_scale
      resized   (ho, wo): cv2.resize's dsize, cvRound(h * scale) (half to even), as prep_image computes it
      padded    (Hp, Wp): resized rounded up to a multiple of `stride` (im_list_to_blob)
      im_info   float32 [3] = (ho, wo, scale), as coco.py:144-147 and cityscapes.py build it from the resized blob
      restored  (out_h, out_w) the label maps are resized back to (upsnet_end2end_test.py:259-266)
      im_post   np.round(im_info[:2] / im_info[2]): the size im_post pastes the masks at (upsnet_end2end_test.py:256)
    The combined panoptic result needs restored == im_post; where they differ the reference fails to broadcast."""
    from .operators import label_restore_geometry
    s = prep_scale(target_size, max_size, h, w)
    ho, wo = int(np.rint(h * s)), int(np.rint(w * s))
    Hp, Wp = -(-ho // stride) * stride, -(-wo // stride) * stride
    info = np.array([ho, wo, s], np.float32)
    restored = label_restore_geometry(info)[3:]
    im_post = tuple(int(v) for v in np.round(info[:2] / info[2]))
    return ImageGeometry(s, (ho, wo), (Hp, Wp), info, restored, im_post)


def scale_for_test_phase(config, dataset):
    """(target_size, max_size) of the reference's test phase.  COCO's loader uses the base get_image_blob, which reads
    config.train.scales / train.max_size even at test time; Cityscapes' override reads config.test.scales /
    test.max_size.  The reference draws one of several scales at random per image, so more than one raises."""
    if dataset not in ("cityscapes", "coco"):
        raise ValueError("dataset must be 'cityscapes' or 'coco', not %r" % (dataset,))
    sec = config.test if dataset == "cityscapes" else config.train
    scales = list(sec.scales)
    if len(scales) != 1:
        raise ValueError("%s test phase: %d scales %s; the reference draws one at random per image, which has no fixed "
                         "geometry" % (dataset, len(scales), scales))
    return scales[0], sec.max_size
