from . import tracking  # noqa: F401
