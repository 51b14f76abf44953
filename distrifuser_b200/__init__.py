"""distrifuser_b200 -- H100-native patch-parallel UNet inference path behind mit-han-lab/distrifuser's API
(DistriConfig / DistriSDXLPipeline / DistriSDPipeline and the Distri*PP module classes)."""
__version__ = "0.1.0"
