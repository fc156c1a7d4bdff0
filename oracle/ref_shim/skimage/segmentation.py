"""Stand-in for skimage.segmentation: find_boundaries is only called by vis_obj_fancy's mask branch, which the fixtures
never take."""


def find_boundaries(*args, **kwargs):
    raise NotImplementedError("skimage stand-in: find_boundaries (vis_obj_fancy's mask branch) is not provided")
