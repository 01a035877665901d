"""Two designed cases of tests/test_gpu_preprocess_edges.py on the CPU executor for the CUDA sources, in the default CPU
tier: both instances of k_project_scatter and the plain-load instance of k_preprocess_tile against the oracle and the
exact model."""
from test_cusim import _child


def test_seam_stencil_case_on_the_cpu_executor():
    """normals, erosion and flood fill across the azimuth seam (one tile)"""
    assert _child(["tests/test_gpu_preprocess_edges.py"], "test_preprocess_case and seam_stencils and 16x5") == 2


def test_tile_case_on_the_cpu_executor():
    """3 x 3 tiles with a partial last tile row and column: winners and stencils across every tile and halo border"""
    assert _child(["tests/test_gpu_preprocess_edges.py"], "test_preprocess_case and tiles and 37x77") == 2
