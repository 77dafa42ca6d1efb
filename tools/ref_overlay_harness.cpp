// tools/ref_overlay_harness.cpp — TEST INFRASTRUCTURE ONLY (never linked into the product). tools/make_overlay_golden.py
// links it with the objects of the unmodified reference and oracle/ref_video_harness.o (make -C oracle ref) into a
// temporary library.
//
// efref_paced_overlay: the instant-decoder pacing of efref_paced_ex (push_video + video_isr, video.cpp:1023-1198) with the
// overlay globals of composite() (video.cpp:839-887) written the way a caller of ef_present_overlay writes them: the
// decoder thread stages push k's command (bitmap / blend / progress, each optional) into a pending slot before it calls
// push_video(k), and the line loop applies the pending slot right before video_isr of every line 0, after the wait for
// _next_frame (so a command staged just before a push is never missed). Tail commands are given per field after the field
// of the last flip and applied at that field's line 0. reset_before[k] != 0: the decoder thread calls video_reset() before
// push_video(k), which leaves the overlay globals alone (video.cpp:1070-1074).
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <chrono>
#include <mutex>
#include <thread>
#include <condition_variable>

#include "player.h"
#undef printf

extern volatile int _line_counter;
extern volatile int _frame_counter;
extern int _line_count, _line_width;
extern int8_t _next_frame, _current_frame;
extern uint32_t _next_frame_time;
void video_reset();
void push_video(Frame* f, int front, int64_t pts, int mode);
extern int16_t _hscroll;
extern int16_t _animate, _animate_index;
extern Frame* _frames;
extern std::mutex _event_guard;
extern std::condition_variable _event_signal;
extern "C" void video_isr(volatile void* vbuf);

namespace {
struct Cmd { int set, blend, progress; const uint8_t* bitmap; };

void load_i420(Frame* f, const uint8_t* s)
{
    for (int y = 0; y < 192; y++, s += 352) memcpy(f->get_y(y), s, 352);
    for (int y = 0; y < 96; y++, s += 176) memcpy(f->get_cr(y), s, 176);
    for (int y = 0; y < 96; y++, s += 176) memcpy(f->get_cb(y), s, 176);
}

void merge(Cmd& into, const Cmd& c)
{
    if (c.set & 1) into.bitmap = c.bitmap;
    if (c.set & 2) into.blend = c.blend;
    if (c.set & 4) into.progress = c.progress;
    into.set |= c.set;
}

void apply(const Cmd& c)
{
    if (c.set & 1) memcpy(_video_composite, c.bitmap, VIDEO_COMPOSITE_WIDTH * VIDEO_COMPOSITE_HEIGHT);
    if (c.set & 2) _video_composite_blend = c.blend;
    if (c.set & 4) _video_composite_progress = c.progress;
}
}  // namespace

extern "C" {

// cmd_* hold n_frames + n_tail entries: push k, then tail field t (the field flip_field[n_frames - 1] + 1 + t); cmd_bitmaps holds
// 1280 bytes per entry. Returns the fields emitted (as efref_paced_ex) and, per field, the blend its overlay lines were drawn with.
long efref_paced_overlay(const uint8_t* i420_frames, int n_frames, const int64_t* pts, const int* modes, const uint8_t* reset_before,
                         int frame_counter0, int max_fields, int tail_fields, const int* cmd_set, const int* cmd_blend, const int* cmd_progress,
                         const uint8_t* cmd_bitmaps, int n_tail, uint16_t* out, uint32_t* flip_field, int* flip_line, int* field_blend)
{
    static Frame* fb = nullptr;
    if (!fb) { fb = new Frame[2]; fb[0].init(); fb[1].init(); }
    video_reset();
    _frames = fb; _current_frame = -1; _next_frame = -1; _next_frame_time = 0;
    _line_counter = 0; _frame_counter = frame_counter0; _hscroll = 0;
    _animate = 0; _animate_index = 0;
    _video_composite_blend = 0; _video_composite_progress = 0;
    memset(_video_composite, 0, sizeof(_video_composite));
    auto cmd = [&](int i) { return Cmd{ cmd_set[i], cmd_blend[i], cmd_progress[i], cmd_bitmaps + (size_t)i * 1280 }; };
    std::mutex guard;
    Cmd pending = { 0, 0, 0, nullptr };
    std::atomic<int> done(0);
    std::thread decoder([&] {
        for (int k = 0; k < n_frames; k++) {
            load_i420(&fb[k & 1], i420_frames + (size_t)k * 101376);
            { std::lock_guard<std::mutex> g(guard); merge(pending, cmd(k)); }
            if (reset_before && reset_before[k]) video_reset();
            push_video(fb, k & 1, pts[k], modes ? modes[k] : 0);
        }
        done = 1;
    });
    uint16_t* lb[2];
    lb[0] = (uint16_t*)calloc(_line_width + 64, 2);
    lb[1] = (uint16_t*)calloc(_line_width + 64, 2);
    const int lines = _line_count, w = _line_width;
    const int overlay_top = (lines == 262 ? 32 : 64) + 192 + 2;
    long fields = 0;
    int flips = 0, tail = -1;
    bool stuck = false;
    while (fields < max_fields && !stuck) {
        for (int l = 0; l < lines && !stuck; l++) {
            const auto t0 = std::chrono::steady_clock::now();
            while (_next_frame == -1 && !done) {
                { std::lock_guard<std::mutex> g(_event_guard); }
                _event_signal.notify_all();
                std::this_thread::yield();
                if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(20)) { stuck = true; break; }
            }
            if (stuck) break;
            if (l == 0) {
                std::lock_guard<std::mutex> g(guard);
                apply(pending);
                pending = Cmd{ 0, 0, 0, nullptr };
                if (done && flips == n_frames) {
                    const uint32_t t = (uint32_t)_frame_counter - (flip_field[n_frames - 1] + 1u);
                    if (t < (uint32_t)n_tail) apply(cmd(n_frames + (int)t));
                }
            }
            if (l == overlay_top && field_blend) field_blend[fields] = _video_composite_blend;
            const int before = _current_frame;
            const uint32_t fc = (uint32_t)_frame_counter;
            video_isr(lb[l & 1]);
            if (_current_frame != before && flips < n_frames) { flip_field[flips] = fc; flip_line[flips] = l; flips++; }
            if (out) memcpy(out + ((size_t)fields * lines + l) * w, lb[l & 1], (size_t)w * 2);
        }
        fields++;
        if (done && _next_frame == -1) {
            if (tail < 0) tail = tail_fields;
            if (tail-- <= 0) break;
        }
    }
    if (!done) {
        _frame_counter = 0x7FFFFFF0;
        for (long g = 0; g < 100000000L && !done; g++) { _line_counter = 0; _next_frame_time = 0; video_isr(lb[0]); std::this_thread::yield(); }
    }
    decoder.join();
    free(lb[0]); free(lb[1]);
    _video_composite_blend = 0;
    return stuck ? -1 : fields;
}

}  // extern "C"
