"""Stand-in for scikit-image (not installed): the sAP toolkit's vis/vis_det_th.py imports skimage.segmentation, whose
find_boundaries only its mask branch calls."""
