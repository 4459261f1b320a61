"""Device-side data layer (SURVEY.md section 8 row f4): see device_pipeline.py."""
from .device_pipeline import (DeviceScanNetAugmentor, DeviceSceneAugmentor, DeviceSunrgbdAugmentor,  # noqa: F401
                              draw_augmentation, draw_augmentation_scannet, draw_augmentation_sunrgbd)
