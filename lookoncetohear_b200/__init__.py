"""lookoncetohear_b200 -- H100 (sm_90a) inference engine for the two networks of
vb000/LookOnceToHear (speaker-conditioned streaming TF-GridNet separator + enrollment embedding
net), behind the reference's own Python call signatures.

    from lookoncetohear_b200 import Net            # drop-in for src.models.tfgridnet_realtime.net.Net
    from lookoncetohear_b200 import EmbedTFGridNet # drop-in for src.models.tfgridnet_orig.tfgridnet.EmbedTFGridNet
    from lookoncetohear_b200 import resample       # for torchaudio.functional.resample(x, orig, new) at its defaults
    from lookoncetohear_b200 import StreamResampler  # the same, pushed a block per tick into a state of slots
    from lookoncetohear_b200 import PacketResampler  # the same, pushed any number of samples per tick
    from lookoncetohear_b200 import HopFifo          # 16 kHz pieces of any length -> separator chunks and hop counts
    from lookoncetohear_b200 import EnrollCapture    # each listener's recent input, kept for EmbedTFGridNet.enroll
    from lookoncetohear_b200 import EnrollJob        # EmbedTFGridNet.enroll_job: an enrollment enqueued in slices
    from lookoncetohear_b200 import TargetHistory    # Net.target_history: block 0's recent output, for Net.join_targets
    from lookoncetohear_b200 import TargetMixer      # each listener's voices and ambient mixture into one row, with fades
    from lookoncetohear_b200 import Limiter          # each listener's output kept under a ceiling, one gain for both ears
    from lookoncetohear_b200 import Leveler          # each voice brought to one loudness, one gain for both ears
    from lookoncetohear_b200 import BandCompressor   # each listener's output fitted to their hearing, per band and ear
    from lookoncetohear_b200 import JitterBuffer     # packets back in sequence order, lost ones concealed

Compute happens only in lib/liblookonce_b200.so (hand-written sm_90a CUDA, C ABI declared in
include/lookonce_b200.h); importing this package never falls back to PyTorch math.
"""
from .embed import EmbedTFGridNet, EnrollJob  # noqa: F401
from .net import Net, SepState, TargetHistory  # noqa: F401
from .render import resample  # noqa: F401
from .stream import BandCompressor, EnrollCapture, HopFifo, JitterBuffer, PacketResampler, Leveler, Limiter, StreamResampler, TargetMixer  # noqa: F401

__all__ = ["Net", "SepState", "TargetHistory", "EmbedTFGridNet", "resample", "StreamResampler", "PacketResampler", "HopFifo",
           "EnrollCapture", "EnrollJob", "TargetMixer", "Limiter", "Leveler",
           "BandCompressor", "JitterBuffer"]
