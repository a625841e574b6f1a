"""contact-human-dynamics, H100-native: batched physics-based trajectory optimisation + foot-contact
classification behind the reference's file boundary.  The directory name carries a hyphen (it mirrors
the reference repo name); import it as `chd` through the repo-root shim `chd.py`."""
from . import io_formats, synth, phys, parallel, contact, prepare, results, kinopt, train  # noqa: F401

__all__ = ["io_formats", "synth", "phys", "parallel", "contact", "prepare", "results", "kinopt", "train"]
