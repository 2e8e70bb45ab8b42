"""open_l2o_b200 - H100-native (sm_90a) engine for the coordinate-wise LSTM learned-optimizer hot path of
Open-L2O's L2O-DM / L2O-RNNProp, behind the reference's MetaOptimizer / networks surface."""
__version__ = "0.1.0"
