"""Import-only stand-in for matplotlib: the reference's core/utils.py imports it for mask drawing, which the I3D /
VFID code never calls."""
