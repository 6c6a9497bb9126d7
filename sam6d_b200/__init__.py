"""sam6d_b200 -- H100-native (sm_90a) implementation of SAM-6D's data-parallel hot path.

    from sam6d_b200.pem import Net                       # drop-in for Pose_Estimation_Model `Net`
    import sam6d_b200.pointnet2_ext as _ext              # drop-in for pointnet2._ext (forward ops)
    from sam6d_b200.ism import PairwiseSimilarity, compute_semantic_score

All compute goes through libsam6d_b200.so (include/sam6d_b200.h); importing this package does not need a GPU, calling
into it does, and there is no CPU / eager fallback.
"""
__version__ = "0.1.0"
