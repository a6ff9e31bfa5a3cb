"""reference vision/data_augmentations.py -> serl_b200."""
from serl_b200.vision.data_augmentations import (adjust_brightness, adjust_contrast, adjust_hue, adjust_saturation,  # noqa: F401
                                                 batched_random_crop, color_transform, gaussian_blur, hsv_to_rgb, random_crop,
                                                 random_flip, rgb_to_hsv, solarize)
