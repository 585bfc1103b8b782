"""The uint8 input edge of SAM encoder distillation (SURVEY.md 8 f3): counterparts of SimpleAICV/interactive_segmentation/
common.py SamResize, SamRandomHorizontalFlip, SamNormalize and SAMBatchCollater.

The image is not resized on the host: its cv2.resize, the flip (which the reference applies after the resize, so the
device mirrors the resized columns) and the float64 (x - mean) / std are recorded and run on the device by
tools.utils.CudaPrefetcher (ops.u8_resize_pad).  Every other key - box, mask, size and the prompts, with their
INTER_NEAREST mask resizes - is computed exactly as the reference computes it."""
import cv2
import numpy as np
import torch

from ..detection.common import GEOM_FLIP, GEOM_OUT_H, GEOM_OUT_W, new_geom, pack_resize_pad


def _record(sample, who):
    rec = sample.get('sam_geom')
    if rec is None:
        raise ValueError(f'{who} follows Uint8SamResize: the sample has no record')
    return rec


class Uint8SamResize:
    """SamResize(resize): box, mask, size and prompts as the reference computes them; the image is kept as uint8 and its
    resize to (resize_h, resize_w) is recorded."""

    def __init__(self, resize=1024):
        self.resize = resize

    def __call__(self, sample):
        image = np.asarray(sample['image'])
        if image.ndim != 3 or image.shape[2] != 3 or sample.get('sam_geom') is not None:
            raise ValueError(f'Uint8SamResize starts the transform list with the decoded [H, W, 3] image, got {image.shape}')
        image = image.astype(np.uint8, copy=False)
        box, mask = sample['box'], sample['mask']
        prompt_point, prompt_box, prompt_mask = sample['prompt_point'], sample['prompt_box'], sample['prompt_mask']

        h, w, _ = image.shape
        factor = self.resize / max(h, w)
        resize_h, resize_w = int(round(h * factor)), int(round(w * factor))
        rec = new_geom(image)
        rec[0][GEOM_OUT_H], rec[0][GEOM_OUT_W] = resize_h, resize_w

        box[0:4] *= factor
        mask = cv2.resize(mask, (resize_w, resize_h), interpolation=cv2.INTER_NEAREST)
        size = np.array([resize_h, resize_w]).astype(np.float32)
        prompt_point[:, 0:2] *= factor
        prompt_box[0:4] *= factor
        prompt_mask = cv2.resize(prompt_mask, (resize_w, resize_h), interpolation=cv2.INTER_NEAREST)

        sample['image'], sample['sam_geom'], sample['box'], sample['mask'], sample['size'] = image, rec, box, mask, size
        sample['prompt_point'], sample['prompt_box'], sample['prompt_mask'] = prompt_point, prompt_box, prompt_mask
        return sample


class Uint8SamRandomHorizontalFlip:
    """SamRandomHorizontalFlip(prob): the same draw, masks, box and prompts; the image's flip toggles the record."""

    def __init__(self, prob=0.5):
        self.prob = prob

    def __call__(self, sample):
        rec = _record(sample, 'Uint8SamRandomHorizontalFlip')
        box, mask = sample['box'], sample['mask']
        prompt_point, prompt_box, prompt_mask = sample['prompt_point'], sample['prompt_box'], sample['prompt_mask']
        if np.random.uniform(0, 1) < self.prob:
            rec[0][GEOM_FLIP] ^= 1
            mask = mask[:, ::-1]
            prompt_mask = prompt_mask[:, ::-1]
            w = int(rec[0][GEOM_OUT_W])
            x1 = box[0].copy()
            x2 = box[2].copy()
            box[0] = w - x2
            box[2] = w - x1
            x1 = prompt_box[0].copy()
            x2 = prompt_box[2].copy()
            prompt_box[0] = w - x2
            prompt_box[2] = w - x1
            for i in range(len(prompt_point)):
                prompt_point[i][0] = w - prompt_point[i][0]
        sample['box'], sample['mask'] = box, mask
        sample['prompt_point'], sample['prompt_box'], sample['prompt_mask'] = prompt_point, prompt_box, prompt_mask
        return sample


class Uint8SamNormalize:
    """SamNormalize(mean, std): recorded; the device computes (x - mean) / std in float64, as numpy does with the
    reference's float64 mean and std, and stores float32."""

    def __init__(self, mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375]):
        self.mean = tuple(float(v) for v in np.array(mean, dtype=np.float64).reshape(3))
        self.std = tuple(float(v) for v in np.array(std, dtype=np.float64).reshape(3))

    def __call__(self, sample):
        _record(sample, 'Uint8SamNormalize')
        sample['sam_norm'] = (self.mean, self.std)
        return sample


class Uint8SAMBatchCollater:
    """SAMBatchCollater(resize) for samples of the Uint8Sam* transforms: 'box', 'mask', 'size', 'prompt_point',
    'prompt_box' and 'prompt_mask' as the reference computes them; the uint8 sources and their records go under
    'resize_pad' (a ResizePadBatch), from which CudaPrefetcher writes the fp32 'image' [B, 3, resize, resize]."""

    def __init__(self, resize, pin_memory=True):
        self.resize = resize
        assert resize % 64 == 0
        self.prompt_mask_size = resize // 4
        self.pin_memory = pin_memory

    def __call__(self, data):
        norms = {s.get('sam_norm') for s in data}
        if len(norms) != 1 or None in norms:
            raise ValueError('Uint8SAMBatchCollater expects every sample to end with the same Uint8SamNormalize')
        boxes = [x['box'] for x in data]
        masks = [x['mask'] for x in data]
        sizes = [x['size'] for x in data]
        prompt_points = [x['prompt_point'] for x in data]
        prompt_boxs = [x['prompt_box'] for x in data]
        prompt_masks = [x['prompt_mask'] for x in data]
        pin = self.pin_memory and torch.cuda.is_available()
        batch = pack_resize_pad(data, 'sam_geom', self.resize, norms.pop(), False, pin)

        input_boxes = []
        for per_box in boxes:
            per_input_box = np.zeros((4), dtype=np.float32)
            per_input_box[0:per_box.shape[0]] = per_box[0:4]
            input_boxes.append(torch.from_numpy(per_input_box))
        input_boxes = torch.stack(input_boxes, dim=0).float()

        input_masks = []
        for per_mask in masks:
            per_input_mask = np.zeros((self.resize, self.resize), dtype=np.float32)
            per_input_mask[0:per_mask.shape[0], 0:per_mask.shape[1]] = per_mask
            input_masks.append(torch.from_numpy(per_input_mask))
        input_masks = torch.stack(input_masks, dim=0).unsqueeze(1).float()

        sizes = np.array(sizes, dtype=np.float32)
        input_prompt_points = torch.stack([torch.from_numpy(p) for p in prompt_points], dim=0).float()
        input_prompt_boxs = torch.stack([torch.from_numpy(p) for p in prompt_boxs], dim=0).float()

        input_prompt_masks = []
        for per_prompt_mask in prompt_masks:
            h, w = per_prompt_mask.shape
            factor = self.prompt_mask_size / max(h, w)
            resize_h, resize_w = int(round(h * factor)), int(round(w * factor))
            per_prompt_mask = cv2.resize(per_prompt_mask, (resize_w, resize_h), interpolation=cv2.INTER_NEAREST)
            per_input_prompt_mask = np.zeros((self.prompt_mask_size, self.prompt_mask_size), dtype=np.float32)
            per_input_prompt_mask[0:per_prompt_mask.shape[0], 0:per_prompt_mask.shape[1]] = per_prompt_mask
            input_prompt_masks.append(torch.from_numpy(per_input_prompt_mask))
        input_prompt_masks = torch.stack(input_prompt_masks, dim=0).unsqueeze(1).float()

        return {
            'resize_pad': batch,
            'box': input_boxes,
            'mask': input_masks,
            'size': sizes,
            'prompt_point': input_prompt_points,
            'prompt_box': input_prompt_boxs,
            'prompt_mask': input_prompt_masks,
        }
