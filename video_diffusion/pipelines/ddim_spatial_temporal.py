from fatezero_b200.pipeline import DDIMSpatioTemporalStableDiffusionPipeline  # noqa: F401
