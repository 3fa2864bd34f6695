"""lamejs_b200 -- host-side mirror of the lamejs `Mp3Encoder` API over the H100-native C-ABI library.

    from lamejs_b200 import Mp3Encoder
    enc = Mp3Encoder(2, 44100, 128)           # new lamejs.Mp3Encoder(channels, sampleRate, kbps)
    mp3 = enc.encodeBuffer(left, right)        # Int16 arrays -> bytes (frames completed by this call)
    mp3 += enc.flush()

(reference: zhuker/lamejs src/js/index.js:66-136).  All computation happens in libmp3b200.so on the GPU; the
module raises if the library or a CUDA device is missing -- there is no CPU fallback.
"""
from .encoder import Mp3Encoder, WavHeader, id3v1_tag, id3v2_tag, ID3_ADD_V2, ID3_V1_ONLY, ID3_V2_ONLY, ID3_SPACE_V1, ID3_PAD_V2, lametag_size, lametag_build, get_vbr_tag, crc16_combine, encode_streams_tagged, debug_music_crc, encode_batch, flush_batch, encode_streams, encode_streams_device, encode_streams_device_tagged, debug_stages, debug_short_units, debug_psy_capture, debug_resample, lib, stream_bytes, stream_frames, granules_per_frame, out_samplerate, RESAMPLE, Mp3B200Error  # noqa: F401
from .encoder import REPLAYGAIN, GAIN_NOT_ENOUGH_SAMPLES, radio_gain, lametag_build_ex, debug_replaygain, encode_streams_replaygain, album_gain  # noqa: F401
from .encoder import DOMAIN_SITES, debug_domain_hits  # noqa: F401
from .encoder import EncodeSession, check_status  # noqa: F401
from .encoder import replay_gain_streams, replay_gain_streams_device, finish_tags_device  # noqa: F401
