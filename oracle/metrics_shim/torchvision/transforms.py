class Compose:
    """transforms.Compose: applies the transforms in order (used by core.utils.to_tensors)."""

    def __init__(self, transforms):
        self.transforms = list(transforms)

    def __call__(self, x):
        for t in self.transforms:
            x = t(x)
        return x
