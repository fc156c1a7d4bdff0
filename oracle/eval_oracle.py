"""CPU restatement of the validation evaluators' ``convert_to_coco_format`` (TEST INFRASTRUCTURE ONLY: imported by tests/
and never by the product).  It follows

  * /root/reference/exps/evaluators/onex_stream_evaluator.py:167-209, twox_stream_evaluator.py:165-217 and
    still_stream_evaluator.py:137-169: per image, ``bboxes /= scale`` (a torch CPU fp32 tensor divided in place by the
    Python float ``scale = min(img_size[0] / h, img_size[1] / w)``), [yolox 0.3.0] ``xyxy2xywh`` (in-place fp32
    subtractions), ``scores = obj * class_conf`` (fp32), ``class_ids[int(cls)]`` and the per-detection frame-id branches,
    whose indentation emits a row only in the final ``else`` of the onex / twox evaluators.

Pinned by tests/test_eval_pipeline.py against the data_lists the unmodified reference methods wrote
(tests/golden/eval_coco_{onex,twox,still}.npz, oracle/make_eval_golden.py)."""
import torch


def output_id(images, img_id, rule):
    """The image id a detection of image ``img_id`` is emitted under, or None when the branches drop it.  ``images`` =
    ``dataset.coco.dataset['images']`` (indexed by id, as the reference indexes it)."""
    img_id = int(img_id)
    if rule == "still":
        return img_id
    if img_id in (15060, 15061):
        return None
    if images[img_id + 1]["fid"] == 0:
        return None
    if rule == "twox" and images[img_id + 2]["fid"] == 0:
        return None
    if images[img_id]["fid"] == 0:               # idd = int(img_id), but nothing is appended in that branch
        return None
    if rule == "twox" and images[img_id]["fid"] == 1:
        return None
    return img_id + (2 if rule == "twox" else 1)


def convert_to_coco_format(outputs, info_imgs, ids, img_size, class_ids, images, rule):
    """the reference method's data_list for one batch: ``outputs`` a list of CPU [n, 7] tensors or None, ``info_imgs``
    (heights, widths), ``ids`` the batch's image ids"""
    data_list = []
    for output, img_h, img_w, img_id in zip(outputs, info_imgs[0], info_imgs[1], ids):
        if output is None:
            continue
        output = output.detach().cpu().clone()
        bboxes = output[:, 0:4]
        scale = min(img_size[0] / float(img_h), img_size[1] / float(img_w))
        bboxes /= scale
        bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 0]
        bboxes[:, 3] = bboxes[:, 3] - bboxes[:, 1]
        cls = output[:, 6]
        scores = output[:, 4] * output[:, 5]
        idd = output_id(images, img_id, rule)
        if idd is None:
            continue
        for ind in range(bboxes.shape[0]):
            data_list.append({"image_id": idd, "category_id": class_ids[int(cls[ind])],
                              "bbox": bboxes[ind].numpy().tolist(), "score": scores[ind].numpy().item(),
                              "segmentation": []})
    return data_list
