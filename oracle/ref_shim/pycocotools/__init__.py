"""Stand-in for the parts of pycocotools (not installed) the sAP forecast script reaches with --no-eval: COCO's image
table, mask.iou for boxes, and a COCOeval that refuses to run."""
