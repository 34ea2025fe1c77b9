"""Executable specification of CMYK and YCCK frames under B200JPG_FLAG_LIBJPEG_TURBO with an output mode (DESIGN §18). TEST-ONLY.

tests/draft_model.py's reconstruction of all four components (libjpeg-turbo's islow or reduced IDCT and its upsampling, no colour
transform) followed by tests/cmyk_model.py's conversion (DESIGN §15). tests/test_turbo_cmyk_cpu.py checks it byte for byte against
Pillow; tests/test_turbo_cmyk.py checks the GPU against it."""
from tests import cmyk_model as km
from tests import draft_model as dm


def reconstruct(coef, width, height, hs, vs, k, space, mode):
    """the image BatchDecoder(reconstruction="libjpeg-turbo", mode=mode) writes for a CMYK / YCCK frame at scale 1/k (k = 1
    undrafted): coef per component [bh, bw, 8, 8] dequantised, width x height the codestream's size, space "CMYK" or "YCCK"
    -> [ceil(H / k), ceil(W / k), 3 or 1] uint8"""
    return km.convert(dm.reconstruct(coef, width, height, hs, vs, k, km.CMYK, color_transform=False), space, mode)
