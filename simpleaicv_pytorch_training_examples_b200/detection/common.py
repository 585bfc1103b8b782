"""The uint8 input edge of the DETR detection recipes (SURVEY.md 8 f3): counterparts of SimpleAICV/detection/common.py
RandomHorizontalFlip, RandomCrop, RandomTranslate, DetectionResize (yolo_style), Normalize and DETRDetectionCollater.

The reference builds every sample in float32 on the host and pads it to resize x resize x 3 (12.6 MB at 1024^2, plus a
1 MB bool mask).  Here the transforms make the reference's np.random draws in its order and update 'annots', 'scale' and
'size' with its float32 numpy expressions; flip and crop stay exact index operations on the uint8 image; the translation
and the resize are only recorded in the sample's 'detection_geom'.  Uint8DETRDetectionCollater packs the uint8 sources
with their records into a ResizePadBatch, and tools.utils.CudaPrefetcher turns it into the reference's fp32 'image' and
bool 'mask' on the device (ops.u8_resize_pad, OpenCV's arithmetic; oracle/detection_input.py restates it)."""
import numpy as np
import torch

# the int32 fields of a sample's 'detection_geom' record and of ResizePadBatch.geom: csrc/capi_input.cu's layout
GEOM_SRC_H, GEOM_SRC_W, GEOM_OUT_H, GEOM_OUT_W, GEOM_FLIP, GEOM_TRANSLATE = range(6)


class ResizePadBatch:
    """The uint8 sources of one DETR or SAM batch and their records, for the device write (ops.u8_resize_pad).

    data uint8 [total]: every sample's [src_h, src_w, 3] source, concatenated (pinned when the collater pins); offsets
    int64 [B]: where image b starts in ``data``; geom int32 [B, 6]: src_h, src_w, out_h, out_w, flip, translate; shift
    float64 [B, 2]: the (tx, ty) of a translated image.  Image b is translated (cv2.warpAffine) when its flag is set,
    resized to out_h x out_w (cv2.resize), mirrored when flip is set, normalised and padded to size x size: x / 255 when
    ``mean`` is None, else (x - mean) / std in float64.  ``with_mask``: the batch also gets DETR's bool padding mask."""

    def __init__(self, data, offsets, geom, shift, size, mean=None, std=None, with_mask=False):
        self.data, self.offsets, self.geom, self.shift = data, offsets, geom, shift
        self.size, self.mean, self.std, self.with_mask = int(size), mean, std, with_mask

    def pin_memory(self):
        """Called by DataLoader(pin_memory=True): only the pixels are copied to the device."""
        self.data = self.data.pin_memory()
        return self


def new_geom(image):
    """The record of an untouched uint8 source: resized to its own size, not flipped, not translated."""
    h, w = image.shape[:2]
    return np.array([h, w, h, w, 0, 0], dtype=np.int32), np.zeros(2, dtype=np.float64)


def pack_resize_pad(data, key, size, norm, with_mask, pin=False):
    """The samples' uint8 sources and ``key`` records (int32 geometry, float64 shift) packed into one ResizePadBatch.
    norm: None for x / 255, else (mean, std).  Raises when a sample has no record or its image does not match it."""
    geoms, shifts, sizes = [], [], []
    for s in data:
        rec = s.get(key)
        if rec is None:
            raise ValueError(f'a sample has no {key!r} record: its transform list must use the Uint8* transforms')
        g, sh = rec
        image = s['image']
        if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.shape != (g[GEOM_SRC_H], g[GEOM_SRC_W], 3):
            raise ValueError(f'a source of {np.shape(image)} does not match its record\'s size {tuple(g[:2])}')
        if g[GEOM_OUT_H] > size or g[GEOM_OUT_W] > size:
            raise ValueError(f'a resized size {tuple(g[2:4])} exceeds the collater\'s {size} x {size}')
        geoms.append(g)
        shifts.append(sh)
        sizes.append(image.size)
    offsets = np.zeros(len(data), dtype=np.int64)
    offsets[1:] = np.cumsum(sizes)[:-1]
    packed = torch.empty(int(sum(sizes)), dtype=torch.uint8, pin_memory=pin)
    flat = packed.numpy()
    for s, off, n in zip(data, offsets, sizes):
        flat[off:off + n].reshape(s['image'].shape)[...] = s['image']
    mean, std = (None, None) if norm is None else norm
    return ResizePadBatch(packed, torch.from_numpy(offsets), torch.from_numpy(np.stack(geoms).astype(np.int32)),
                          torch.from_numpy(np.stack(shifts).astype(np.float64)), size, mean, std, with_mask)


def _u8_sample(sample, who):
    """(uint8 image, record) of a sample, starting the record (and converting the dataset's integer-valued float32 image
    to uint8) at the first Uint8* transform."""
    rec = sample.get('detection_geom')
    image = sample['image']
    if rec is None:
        image = np.asarray(image)
        if image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f'{who} expects the decoded [H, W, 3] image, got {image.dtype} {image.shape}')
        image = image.astype(np.uint8, copy=False)
        rec = sample['detection_geom'] = new_geom(image)
        sample['image'] = image
    return image, rec


def _exact(rec, who):
    g = rec[0]
    if g[GEOM_TRANSLATE] or (g[GEOM_OUT_H], g[GEOM_OUT_W]) != (g[GEOM_SRC_H], g[GEOM_SRC_W]):
        raise ValueError(f'{who} after Uint8RandomTranslate or Uint8DetectionResize is not implemented: it would have to '
                         'act on the recorded image')


class Uint8RandomHorizontalFlip:
    """RandomHorizontalFlip(prob) on the uint8 image: the same draw (none when 'annots' is empty), the same annots."""

    def __init__(self, prob=0.5):
        self.prob = prob

    def __call__(self, sample):
        image, rec = _u8_sample(sample, 'Uint8RandomHorizontalFlip')
        annots = sample['annots']
        if annots.shape[0] == 0:
            return sample
        _exact(rec, 'Uint8RandomHorizontalFlip')
        if np.random.uniform(0, 1) < self.prob:
            image = image[:, ::-1, :]
            _, w, _ = image.shape
            x1 = annots[:, 0].copy()
            x2 = annots[:, 2].copy()
            annots[:, 0] = w - x2
            annots[:, 2] = w - x1
            sample['size'] = np.array([image.shape[0], image.shape[1]]).astype(np.float32)
            sample['image'] = image
        return sample


class Uint8RandomCrop:
    """RandomCrop(prob) on the uint8 image: the same draws, the same slice, annots and size."""

    def __init__(self, prob=0.5):
        self.prob = prob

    def __call__(self, sample):
        image, rec = _u8_sample(sample, 'Uint8RandomCrop')
        annots = sample['annots']
        if annots.shape[0] == 0:
            return sample
        _exact(rec, 'Uint8RandomCrop')
        if np.random.uniform(0, 1) < self.prob:
            h, w, _ = image.shape
            max_bbox = np.concatenate([np.min(annots[:, 0:2], axis=0), np.max(annots[:, 2:4], axis=0)], axis=-1)
            max_left_trans, max_up_trans = max_bbox[0], max_bbox[1]
            max_right_trans, max_down_trans = w - max_bbox[2], h - max_bbox[3]
            crop_xmin = max(0, int(max_bbox[0] - np.random.uniform(0, max_left_trans)))
            crop_ymin = max(0, int(max_bbox[1] - np.random.uniform(0, max_up_trans)))
            crop_xmax = min(w, int(max_bbox[2] + np.random.uniform(0, max_right_trans)))
            crop_ymax = min(h, int(max_bbox[3] + np.random.uniform(0, max_down_trans)))
            image = image[crop_ymin:crop_ymax, crop_xmin:crop_xmax]
            annots[:, [0, 2]] = annots[:, [0, 2]] - crop_xmin
            annots[:, [1, 3]] = annots[:, [1, 3]] - crop_ymin
            sample['size'] = np.array([image.shape[0], image.shape[1]]).astype(np.float32)
            sample['image'] = image
            sample['detection_geom'] = new_geom(image)
        return sample


class Uint8RandomTranslate:
    """RandomTranslate(prob): the same draws and annots; the cv2.warpAffine translation by (tx, ty) is recorded and run on
    the device."""

    def __init__(self, prob=0.5):
        self.prob = prob

    def __call__(self, sample):
        image, rec = _u8_sample(sample, 'Uint8RandomTranslate')
        annots = sample['annots']
        if annots.shape[0] == 0:
            return sample
        _exact(rec, 'Uint8RandomTranslate')
        if np.random.uniform(0, 1) < self.prob:
            h, w, _ = image.shape
            max_bbox = np.concatenate([np.min(annots[:, 0:2], axis=0), np.max(annots[:, 2:4], axis=0)], axis=-1)
            max_left_trans, max_up_trans = max_bbox[0], max_bbox[1]
            max_right_trans, max_down_trans = w - max_bbox[2], h - max_bbox[3]
            tx = np.random.uniform(-(max_left_trans - 1), (max_right_trans - 1))
            ty = np.random.uniform(-(max_up_trans - 1), (max_down_trans - 1))
            annots[:, [0, 2]] = annots[:, [0, 2]] + tx
            annots[:, [1, 3]] = annots[:, [1, 3]] + ty
            rec[0][GEOM_TRANSLATE] = 1
            rec[1][:] = (tx, ty)
            sample['size'] = np.array([h, w]).astype(np.float32)
        return sample


class Uint8DetectionResize:
    """DetectionResize with resize_type='yolo_style': the same multi-scale draw, factor, annots, scale and size; the
    cv2.resize to (resize_h, resize_w) is recorded and run on the device.  retina_style is not implemented."""

    def __init__(self, resize=800, stride=32, resize_type='retina_style', multi_scale=False, multi_scale_range=[0.8, 1.0]):
        assert resize_type in ['retina_style', 'yolo_style']
        if resize_type != 'yolo_style':
            raise NotImplementedError(f'Uint8DetectionResize resize_type={resize_type!r}: only yolo_style (the DETR '
                                      'recipes\') is implemented')
        assert 0.0 < multi_scale_range[0] <= 1.0
        assert 0.0 < multi_scale_range[1] <= 1.0
        assert multi_scale_range[0] <= multi_scale_range[1]
        self.resize, self.stride, self.multi_scale, self.multi_scale_range = resize, stride, multi_scale, multi_scale_range

    def __call__(self, sample):
        image, rec = _u8_sample(sample, 'Uint8DetectionResize')
        annots, scale = sample['annots'], sample['scale']
        h, w, _ = image.shape
        if self.multi_scale:
            scale_range = [int(self.multi_scale_range[0] * self.resize), int(self.multi_scale_range[1] * self.resize)]
            resize_list = [i // self.stride * self.stride for i in range(scale_range[0], scale_range[1] + self.stride)]
            resize_list = list(set(resize_list))
            random_idx = np.random.randint(0, len(resize_list))
            final_resize = resize_list[random_idx]
        else:
            final_resize = self.resize
        factor = final_resize / max(h, w)
        resize_h, resize_w = int(round(h * factor)), int(round(w * factor))
        if resize_h < 1 or resize_w < 1:
            raise ValueError(f'Uint8DetectionResize: a {h} x {w} image resizes to {resize_h} x {resize_w}')
        rec[0][GEOM_OUT_H], rec[0][GEOM_OUT_W] = resize_h, resize_w
        factor = np.float32(factor)
        annots[:, :4] *= factor
        scale *= factor
        sample['annots'], sample['scale'] = annots, scale
        sample['size'] = np.array([resize_h, resize_w]).astype(np.float32)
        return sample


class Uint8Normalize:
    """Normalize (image / 255.): recorded; the device divides in float32, as numpy does for the float32 image."""

    def __call__(self, sample):
        _u8_sample(sample, 'Uint8Normalize')
        sample['detection_norm'] = True
        return sample


class Uint8DETRDetectionCollater:
    """DETRDetectionCollater for samples of the Uint8* transforms: 'annots', 'scaled_annots', 'scale', 'size' and
    'scaled_size' as the reference computes them; the uint8 sources and their records go under 'resize_pad' (a
    ResizePadBatch), from which CudaPrefetcher writes the fp32 'image' [B, 3, resize, resize] and the bool 'mask'."""

    def __init__(self, resize=800, resize_type='yolo_style', max_annots_num=100, pin_memory=True):
        assert resize_type in ['retina_style', 'yolo_style']
        self.resize = resize
        if resize_type == 'retina_style':
            self.resize = int(round(self.resize * 1333. / 800))
        self.max_annots_num = max_annots_num
        self.pin_memory = pin_memory

    def __call__(self, data):
        if not all(s.get('detection_norm') for s in data):
            raise ValueError('Uint8DETRDetectionCollater expects every sample to end with Uint8Normalize')
        annots = [s['annots'] for s in data]
        scales = [s['scale'] for s in data]
        sizes = [s['size'] for s in data]
        pin = self.pin_memory and torch.cuda.is_available()
        batch = pack_resize_pad(data, 'detection_geom', self.resize, None, True, pin)
        scaled_sizes = [[int(g[GEOM_OUT_H]), int(g[GEOM_OUT_W])] for g in batch.geom.numpy()]

        input_annots = np.ones((len(annots), self.max_annots_num, 5), dtype=np.float32) * (-1)
        for i, annot in enumerate(annots):
            if annot.shape[0] > 0:
                input_annots[i, :annot.shape[0], :] = annot
        input_annots = torch.from_numpy(input_annots).float()

        scaled_annots = np.ones((len(annots), self.max_annots_num, 5), dtype=np.float32) * (-1)
        for i, annot in enumerate(annots):
            h, w = scaled_sizes[i][0], scaled_sizes[i][1]
            per_image_size = np.array([w, h, w, h], dtype=np.float32)
            if annot.shape[0] > 0:
                annot_center = (annot[:, 0:2] + annot[:, 2:4]) / 2
                annot_wh = annot[:, 2:4] - annot[:, 0:2]
                annot_label = annot[:, 4:5]
                annot_cxcywh = np.concatenate([annot_center, annot_wh], axis=1)
                annot_cxcywh = annot_cxcywh / per_image_size
                annot_cxcywh = np.concatenate([annot_cxcywh, annot_label], axis=1)
                scaled_annots[i, :annot_cxcywh.shape[0], :] = annot_cxcywh
        scaled_annots = torch.from_numpy(scaled_annots).float()

        return {
            'resize_pad': batch,
            'annots': input_annots,
            'scale': np.array(scales, dtype=np.float32),
            'size': np.array(sizes, dtype=np.float32),
            'scaled_annots': scaled_annots,
            'scaled_size': np.array(scaled_sizes, dtype=np.float32),
        }
