// tools/ref_restart_harness.cpp — TEST INFRASTRUCTURE ONLY (never linked into the product). tools/make_restart_golden.py
// builds it against the objects of the unmodified reference (make -C oracle ref) in a temporary directory, in two forms.
//
// -DEFREF_RESTART_DECODER: a CLI over the reference's decoder thread with player.cpp compiled with the audio harness's hooks
// (oracle/_ref/player_aud.o: push_audio / push_video call out here). It plays programs one after the other the way the
// reference's player restarts its decoder (espflix.cpp:787-797, 1060-1068): every program ends with the end-of-stream buffer
// (the decoder pauses at the sequence end code, player.cpp:1322-1325); before the next one the player calls
// MpegDecoder::reset() and video_reset() (player.cpp:439-453, video.cpp:1070-1074) and lets the decoder run again. Audio is
// drained at once as in oracle/ref_audio_harness.cpp (decode_audio() after every push_audio(), write_pcm_16() ->
// pdm_second_order() from the sketch). After the last program the last picture is flushed (flush_picture(1)).
//   efref_restart <out.bin> <a.ts> [<b.ts> ...]
//   out = i64 n_programs, i64 n_pushes, i64 n_pcm, then per program i64 pushes / pcm samples / get_pts() at its end,
//         i64 pts of every push, int16 pcm[n_pcm], uint16 pdm[2 n_pcm]
//
// -DEFREF_RESTART_PACED: efref_restart_hook, linked with tools/ref_overlay_harness.cpp compiled with
// -Dvideo_reset=efref_restart_hook, so that its reset_before[k] runs video_reset() (op 1) or video_pause(0) (op 2) as chosen by
// efref_restart_op() for the whole run; the harness's own reset at the start of a run stays video_reset().
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include <chrono>
#include <string>
#include <thread>
#include <vector>

#include "player.h"
#undef printf

#ifdef EFREF_RESTART_PACED
void video_reset();
void video_pause(int p);
static int g_op = 1, g_calls = 0;
void efref_restart_hook()
{
    if (g_calls++ == 0 || g_op == 1) video_reset();
    else video_pause(0);
}
extern "C" void efref_restart_op(int op) { g_op = op; g_calls = 0; }
#endif

#ifdef EFREF_RESTART_DECODER
#include "_ref/pdm_extract.inc"      // void pdm_second_order(uint16_t* dst, const int16_t* src, int len, int32_t a1, int a2)

extern "C" int efref_putchar(int c) { (void)c; return c; }
std::string to_string(int i) { return std::to_string(i); }
void video_init_hw(int, int) {}
void ir_sample() {}

static std::vector<int16_t> g_pcm;
static std::vector<uint16_t> g_pdm;
static std::vector<int64_t> g_push;

void push_audio(const uint8_t* data, int len, int64_t pts, bool pes_complete);   // video.cpp:1007 (the real one)
int decode_audio();                                                              // video.cpp:964
void video_reset();                                                              // video.cpp:1070

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
    push_audio(data, len, pts, pes_complete);
    while (decode_audio()) {}
}
void efref_hook_push_video(Frame*, int, int64_t pts, int) { g_push.push_back(pts); }

static std::vector<uint8_t> load(const char* path)
{
    std::vector<uint8_t> v;
    FILE* f = fopen(path, "rb");
    if (!f) { perror(path); _exit(2); }
    uint8_t tmp[65536]; size_t n;
    while ((n = fread(tmp, 1, sizeof(tmp), f)) > 0) v.insert(v.end(), tmp, tmp + n);
    fclose(f);
    return v;
}

static void wait_paused()
{
    while (!(get_events() & DECODER_PAUSED)) std::this_thread::sleep_for(std::chrono::microseconds(200));
}

int main(int argc, char** argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s out.bin a.ts [b.ts ...]\n", argv[0]); return 2; }
    video_init(1);                    // sbc_init(&_sbc), video.cpp:595
    Frame* fb = new Frame[2];
    fb[0].init(); fb[1].init();
    MpegDecoder* dec = new MpegDecoder(&fb[0], &fb[1]);
    clear_events(DECODER_PAUSED);
    set_events(DECODER_RUN);
    std::thread* th = new std::thread([dec] { dec->run(); });
    std::vector<int64_t> ends;
    const int n_prog = argc - 2;
    for (int p = 0; p < n_prog; p++) {
        if (p) {                      // play(): _decoder.reset(); video_reset(); set_events(DECODER_RUN)
            dec->reset();
            video_reset();
            clear_events(DECODER_PAUSED);
            set_events(DECODER_RUN);
        }
        const std::vector<uint8_t> ts = load(argv[2 + p]);
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
        wait_paused();
        ends.push_back((int64_t)g_push.size());
        ends.push_back((int64_t)g_pcm.size());
        ends.push_back(dec->get_pts());
    }
    dec->flush_picture(1);
    th->detach();

    FILE* o = fopen(argv[1], "wb");
    if (!o) { perror(argv[1]); _exit(2); }
    const int64_t hdr[3] = { n_prog, (int64_t)g_push.size(), (int64_t)g_pcm.size() };
    fwrite(hdr, 8, 3, o);
    fwrite(ends.data(), 8, ends.size(), o);
    fwrite(g_push.data(), 8, g_push.size(), o);
    fwrite(g_pcm.data(), 2, g_pcm.size(), o);
    fwrite(g_pdm.data(), 2, g_pdm.size(), o);
    fclose(o);
    _exit(0);
}
#endif
