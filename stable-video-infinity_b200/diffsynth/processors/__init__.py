"""Video processors with the reference's in-memory interface (diffsynth/processors): PIL frames in, PIL frames out."""
