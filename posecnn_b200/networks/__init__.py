# mirrors lib/networks/__init__.py of the reference, which exports each network class under its module name
from .vgg16_det import vgg16_det  # noqa: F401
