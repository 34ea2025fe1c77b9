"""Flips of BatchDecoder(hflip=..., vflip=...) / b200jpg_batch_create_flip (DESIGN §21): the numpy definition, the dihedral
product of a flip and an Exif orientation that the plan of a frame without a size takes, and the mirrored crop rectangle."""
import numpy as np

H, V = 1, 2  # B200JPG_FLIP_H, B200JPG_FLIP_V

# ORIENTATION[o - 1][f]: the orientation that writes flip(orient(D, o), f) (abi.cpp: kFlipOrientation)
ORIENTATION = [[1, 2, 4, 3], [2, 1, 3, 4], [3, 4, 2, 1], [4, 3, 1, 2], [5, 6, 8, 7], [6, 5, 7, 8], [7, 8, 6, 5], [8, 7, 5, 6]]


def flip(a, f):
    """O ([h, w, ...], or a list of planes each flipped at its own extent) -> O[:, ::-1] for H, O[::-1] for V, both for H | V"""
    if a is None:
        return None
    if isinstance(a, list):
        return [flip(p, f) for p in a]
    if f & H:
        a = a[:, ::-1]
    if f & V:
        a = a[::-1]
    return np.ascontiguousarray(a)


def flip_rect(r, f, w, h):
    """the rectangle (x, y, width, height) of a w x h image as the rectangle of its flip that holds the same samples"""
    x, y, rw, rh = r
    return (w - x - rw if f & H else x, h - y - rh if f & V else y, rw, rh)
