"""H100-native drop-in for LongVideoGAN's ``torch_utils.ops`` operator set."""
