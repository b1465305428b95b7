"""spectralcluster_b200: the SpectralClusterer.predict() hot path of wq2012/SpectralCluster,
built from scratch for NVIDIA H100 (sm_90a).

The package-level names mirror the reference's import surface for that path
(/root/reference/spectralcluster/__init__.py:14-43): users switch by changing the import.
Every module of the reference package has its mirror here; DESIGN.md section 1 says which parts
run on the device and which are host logic around it.
"""

from . import (autotune, configs, constraint, custom_distance_kmeans, fallback_clusterer,
               laplacian, multi_stage_clusterer, naive_clusterer, refinement, spectral_clusterer,
               utils)

__version__ = "0.1.0"

# public name -> defining submodule
_EXPORTS = {
    autotune: ("AutoTune", "AutoTuneProxy"),
    constraint: ("ConstraintOptions", "ConstraintName", "ConstraintMatrix", "IntegrationType"),
    naive_clusterer: ("NaiveClusterer",),
    fallback_clusterer: ("FallbackOptions", "SingleClusterCondition", "FallbackClustererType"),
    laplacian: ("LaplacianType",),
    refinement: ("RefinementName", "RefinementOptions", "ThresholdType", "SymmetrizeType"),
    spectral_clusterer: ("SpectralClusterer",),
    utils: ("EigenGapType",),
    configs: ("ICASSP2018_REFINEMENT_SEQUENCE", "TURNTODIARIZE_REFINEMENT_SEQUENCE"),
    multi_stage_clusterer: ("Deflicker", "MultiStageClusterer"),
}
for _module, _names in _EXPORTS.items():
  for _name in _names:
    globals()[_name] = getattr(_module, _name)

__all__ = sorted(n for names in _EXPORTS.values() for n in names) + [
    "autotune", "configs", "constraint", "custom_distance_kmeans", "fallback_clusterer", "laplacian",
    "multi_stage_clusterer", "naive_clusterer", "refinement", "spectral_clusterer", "utils"]
del _module, _names, _name
