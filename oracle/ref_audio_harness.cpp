// oracle/ref_audio_harness.cpp — TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// The reference's audio path, unmodified, as a CPU checker (SURVEY.md 8f-3): MpegDecoder::more()/demux()
// (player.cpp:381-493) route the payload of PID 0x101 / 0x102 to push_audio() (video.cpp:1007), decode_audio()
// (video.cpp:964) runs sbc_decoder() (sbc_decoder.cpp:343) frame by frame and hands 128 PCM samples to
// write_pcm_16(), which on the device runs pdm_second_order() (espflix.ino:73). Here:
//   * player.cpp is compiled a second time with -Dpush_audio=efref_hook_push_audio -Dpush_video=efref_hook_push_video
//     (oracle/Makefile): the hooks below record what the demux pushes, call the REAL push_audio of video.cpp and drain
//     the 4 KB ring with the REAL decode_audio at once (the "instant audio thread" model: no overflow, no pacing);
//   * write_pcm_16 (an ESP-only hook, espflix.ino:123) records the PCM and runs pdm_second_order, whose text the
//     Makefile extracts from espflix.ino into _ref/pdm_extract.inc at build time (the sketch itself needs the Arduino SDK).
// CLI (one run per process: decoder scratch, _sbc and the modulator state are process globals):
//   efref_audio <in.ts> <out.bin>       out = u64 es_bytes, u64 pcm_samples, es bytes, pcm int16[], pdm uint16[2*pcm]
//   efref_audio -es <in.sbc> <out.bin>  the SBC bytes handed to the REAL push_audio in one call, then decode_audio until
//                                       it stops: every byte a frame's bit loader reads is in the ring when the frame
//                                       is decoded (a stream of at most 4 KB - 264 bytes never wraps the ring, and the
//                                       bytes after its end are the ring's initial zeros); same output file
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include <string>
#include <thread>
#include <chrono>
#include <vector>

#include "player.h"
#undef printf

#include "_ref/pdm_extract.inc"      // void pdm_second_order(uint16_t* dst, const int16_t* src, int len, int32_t a1, int a2)

extern "C" int efref_putchar(int c) { (void)c; return c; }
std::string to_string(int i) { return std::to_string(i); }
void video_init_hw(int, int) {}
void ir_sample() {}

static std::vector<uint8_t> g_es;
static std::vector<int16_t> g_pcm;
static std::vector<uint16_t> g_pdm;

void push_audio(const uint8_t* data, int len, int64_t pts, bool pes_complete);   // video.cpp:1007 (the real one)
int decode_audio();                                                              // video.cpp:964

void write_pcm_16(const int16_t* s, int n, int channels)
{
    (void)channels;
    if (!s) return;
    g_pcm.insert(g_pcm.end(), s, s + n);
    std::vector<uint16_t> out((size_t)n * 2);
    pdm_second_order(out.data(), s, n);
    g_pdm.insert(g_pdm.end(), out.begin(), out.end());
}

void efref_hook_push_audio(const uint8_t* data, int len, int64_t pts, bool pes_complete)
{
    g_es.insert(g_es.end(), data, data + len);
    push_audio(data, len, pts, pes_complete);
    while (decode_audio()) {}
}
void efref_hook_push_video(Frame*, int, int64_t, int) {}

static void write_out(const char* path)
{
    FILE* o = fopen(path, "wb");
    if (!o) { perror(path); _exit(2); }
    uint64_t hdr[2] = { g_es.size(), g_pcm.size() };
    fwrite(hdr, 8, 2, o);
    fwrite(g_es.data(), 1, g_es.size(), o);
    fwrite(g_pcm.data(), 2, g_pcm.size(), o);
    fwrite(g_pdm.data(), 2, g_pdm.size(), o);
    fclose(o);
    fprintf(stdout, "{\"es_bytes\": %zu, \"pcm_samples\": %zu, \"pdm_words\": %zu}\n", g_es.size(), g_pcm.size(), g_pdm.size());
    fflush(stdout);
}

int main(int argc, char** argv)
{
    const bool es_mode = argc >= 4 && !strcmp(argv[1], "-es");
    if (argc < 3) { fprintf(stderr, "usage: %s [-es] in.ts|in.sbc out.bin\n", argv[0]); return 2; }
    const char* in = argv[es_mode ? 2 : 1];
    const char* out = argv[es_mode ? 3 : 2];
    FILE* f = fopen(in, "rb");
    if (!f) { perror(in); return 2; }
    std::vector<uint8_t> ts;
    uint8_t tmp[65536]; size_t n;
    while ((n = fread(tmp, 1, sizeof(tmp), f)) > 0) ts.insert(ts.end(), tmp, tmp + n);
    fclose(f);

    video_init(1);                    // sbc_init(&_sbc), video.cpp:595
    if (es_mode) {
        if (ts.size() + 264 > 4096) { fprintf(stderr, "%s: more than 4 KB - 264 bytes\n", in); return 2; }
        g_es = ts;
        if (!ts.empty()) push_audio(ts.data(), (int)ts.size(), 0, true);
        while (decode_audio()) {}
        write_out(out);
        _exit(0);
    }
    Frame* fb = new Frame[2];
    fb[0].init(); fb[1].init();
    MpegDecoder* dec = new MpegDecoder(&fb[0], &fb[1]);
    clear_events(DECODER_PAUSED);
    set_events(DECODER_RUN);
    std::thread* th = new std::thread([dec] { dec->run(); });
    size_t pos = 0;
    while (pos + 188 <= ts.size()) {
        Buffer* b = dec->pop_empty();
        if (!b) continue;
        size_t k = ts.size() - pos;
        if (k > sizeof(b->data)) k = sizeof(b->data);
        k -= k % 188;
        memcpy(b->data, ts.data() + pos, k);
        b->len = (uint32_t)k;
        pos += k;
        dec->push_full(b);
    }
    Buffer* b;
    while (!(b = dec->pop_empty())) {}
    b->len = 0;
    dec->push_full(b);
    while (!(get_events() & DECODER_PAUSED)) std::this_thread::sleep_for(std::chrono::microseconds(200));
    th->detach();

    write_out(out);
    _exit(0);
}
