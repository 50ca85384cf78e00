"""voxelmorph.generators (reference voxelmorph/generators.py) -> voxelmorph_b200.generators."""
from voxelmorph_b200.generators import *          # noqa: F401,F403
from voxelmorph_b200.generators import load_volfile, volgen, scan_to_scan, scan_to_atlas, semisupervised  # noqa: F401
from voxelmorph_b200.generators import template_creation, conditional_template_creation, hypermorph  # noqa: F401
from voxelmorph_b200.generators import surf_semisupervised  # noqa: F401
