"""selfocc_b200 -- Hopper (H100, sm_90a) implementation of SelfOcc's two hot paths:
image -> tri-plane lifting (multi-scale deformable attention) and the SDF volume-render head,
behind the reference's registry/module API.  See DESIGN.md."""
__version__ = '0.1.0'
