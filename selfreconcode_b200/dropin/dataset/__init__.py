from .dataset import SceneDataset, RandomSampler, ClipSampler, ShardedSampler, getDatasetAndLoader, write_sequence, \
    FrameLoader, FrameStore, frame_store, pack_mask
