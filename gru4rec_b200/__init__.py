"""gru4rec_b200 -- H100-native GRU4Rec training step behind the reference's GRU4Rec class surface."""
