from elasticdl_b200.preprocessing.layers import (  # noqa: F401
    ConcatenateWithOffset,
    Discretization,
    FeatureTransform,
    Hashing,
    IndexLookup,
    LogRound,
    Normalizer,
    RoundIdentity,
    build_vocab_table,
    encode_strings,
    read_vocabulary_file,
)
