"""Import-only stand-in for torchvision: the reference's core/utils.py imports ``transforms`` for ``Compose``."""
