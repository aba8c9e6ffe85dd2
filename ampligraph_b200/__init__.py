"""ampligraph_b200 -- H100-native (sm_90a) replacement for AmpliGraph's training /
ranking hot path behind the reference's ScoringBasedEmbeddingModel API.

    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel

Importing the package never touches CUDA; the first model/engine construction
dlopens libkge_b200.so and needs an H100 (sm_90).
"""
__version__ = "0.1.0"
