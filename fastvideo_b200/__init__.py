"""fastvideo_b200: H100 (sm_90a) implementation of FastVideo's Wan DiT denoising hot path and Wan VAE
decode, behind the reference's attention-backend / layer-operator interfaces. See DESIGN.md."""
__version__ = "0.1.0"
