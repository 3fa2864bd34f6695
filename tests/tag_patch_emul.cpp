/* tag_patch_emul.cpp -- the data-dependent bytes of a tag frame on the CPU (lamejs_b200/csrc/k_tag.cuh compiled by g++): the
 * __host__ __device__ functions k_tag_finish completes a template frame with are the ones mp3_tag_frame ends in, so patching
 * a frame here must give what the library builds directly.  TEST INFRASTRUCTURE (tests/test_tag_patch_cpu.py). */
#include "../lamejs_b200/csrc/k_tag.cuh"

extern "C" {

int emul_radio_gain(double title_db) { return mp3_radio_gain(title_db); }
int emul_radio_gain_field(int radio_gain) { return mp3_radio_gain_field(radio_gain); }
int emul_head_bytes(int sideinfo_len) { Mp3TagParams p = {}; p.sideinfo_len = sideinfo_len; return mp3_tag_head_bytes(p); }

/* what thread 0 of k_tag_finish does to the staged head of a frame; analysed == 0: the field stays 0 */
void emul_patch(uint8_t* frame, int sideinfo_len, unsigned music_crc, int analysed, double title_db) {
  Mp3TagParams p = {};
  p.sideinfo_len = sideinfo_len;
  mp3_tag_patch(frame, p, music_crc & 0xffffu, analysed ? mp3_radio_gain_field(mp3_radio_gain(title_db)) : 0);
}

}
