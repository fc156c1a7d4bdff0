import json


class COCO:
    """the annotation file's ``dataset`` and ``imgs`` (id -> image, in the order of dataset['images'])"""

    def __init__(self, annotation_file=None):
        self.dataset, self.imgs = {}, {}
        if annotation_file is not None:
            with open(annotation_file) as f:
                self.dataset = json.load(f)
            for img in self.dataset.get("images", []):
                self.imgs[img["id"]] = img
