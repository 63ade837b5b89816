"""meshdiffusion_b200: H100-native (sm_90a) implementation of MeshDiffusion's score-network / sampler / marching-tet hot path."""
__version__ = "0.1.0"
