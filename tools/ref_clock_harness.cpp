// tools/ref_clock_harness.cpp — the reference's own ESPFlix::update_progress() and show_time() (espflix.cpp:163-174, 862-874),
// compiled from the UNMODIFIED espflix.cpp, for tools/make_clock_golden.py. TEST INFRASTRUCTURE ONLY.
//
// espflix.cpp is included whole under `#define class struct`, so the harness reaches ESPFlix's private members (_nav, _speed,
// _state, _info, _last_seconds). Every standard header is included first, so the macro touches only the reference's own text.
// The player, display, streamer, events, Wi-Fi, key and storage symbols it references are stubbed below; player.o and video.o are
// not linked. MpegDecoder::get_pts() returns g_pts, the value the caller hands over. _video_composite is the head of a larger
// buffer: show_time() writes the spill of text wider than 80 pixels past row 15, outside the 1,280 bytes that are compared.
#include <math.h>
#include <pthread.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <functional>
#include <list>
#include <map>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

#define class struct
#include "espflix.cpp"
#undef class

static int64_t g_pts = -1;
extern "C" { uint8_t efref_composite_area[VIDEO_COMPOSITE_HEIGHT * VIDEO_COMPOSITE_WIDTH + 4096]; }
extern uint8_t _video_composite[VIDEO_COMPOSITE_HEIGHT * VIDEO_COMPOSITE_WIDTH] __attribute__((alias("efref_composite_area")));
int _video_composite_blend;
int _video_composite_progress;

// ---- stubs: nothing below is reached by update_progress() / show_time() except get_pts() ----
void Frame::init() {}
uint8_t* Frame::get_y(int) { return efref_composite_area; }
void Frame::erase() {}
MpegDecoder::MpegDecoder(Frame*, Frame*) {}
void MpegDecoder::flush_picture(int) {}
int64_t MpegDecoder::get_pts() { return g_pts; }
Buffer* MpegDecoder::pop_empty() { return nullptr; }
void MpegDecoder::push_full(Buffer*) {}
void MpegDecoder::reset() {}
void MpegDecoder::run() {}
int Streamer::get(const char*, uint32_t, uint32_t) { return -1; }
void Streamer::get_rom(const uint8_t*, int) {}
int Streamer::get_url(const char*, std::vector<uint8_t>&, uint32_t, uint32_t) { return -1; }
ssize_t Streamer::read(uint8_t*, uint32_t, uint32_t*) { return -1; }
extern "C" void audio_thread(void*) {}
void beep() {}
void clear_events(int) {}
void set_events(int) {}
void wait_events(int) {}
int get_events() { return 0; }
void up_key() {}
void down_key() {}
int get_nec() { return 0; }
int64_t nv_read(const char*) { return 0; }
void nv_write(const char*, int64_t) {}
int printf_nano(const char*, ...) { return 0; }
void push_video(Frame*, int, int64_t, int) {}
int stack() { return 0; }
void start_thread(TaskFunction_t, void*, int) {}
void video_init(int) {}
void video_pause(int) {}
void video_reset() {}
void wifi_disconnect() {}
void wifi_join(const char*, const char*) {}
std::map<std::string, int>& wifi_list() { static std::map<std::string, int> m; return m; }
std::string wifi_ssid() { return std::string(); }
WiFiState wifi_state() { return NONE; }

static ESPFlix* player()
{
    static ESPFlix* p = nullptr;
    if (!p) {
        p = new ESPFlix(1);
        p->_info.resize(1);
    }
    return p;
}

extern "C" {

// one update_progress() with get_pts() = pts on title 0 whose video.idx header is hdr (104 bytes); zero_last first sets
// _last_seconds = 0 as play_pause() does. Out: the bitmap (1,280 bytes), _video_composite_progress and _last_seconds.
void efref_update_progress(const uint8_t* hdr, int speed, int paused, int zero_last, int64_t pts, uint8_t* bitmap, int* progress,
                           int64_t* last_seconds)
{
    ESPFlix* p = player();
    static_assert(sizeof(p->_info[0].idx) == 104, "idx_hdr");
    memcpy(&p->_info[0].idx, hdr, 104);
    p->_nav = 0;
    p->_speed = speed;
    p->_state = paused ? ESPFlix::PAUSED : ESPFlix::PLAYING;
    if (zero_last) p->_last_seconds = 0;
    g_pts = pts;
    p->update_progress();
    memcpy(bitmap, _video_composite, VIDEO_COMPOSITE_HEIGHT * VIDEO_COMPOSITE_WIDTH);
    *progress = _video_composite_progress;
    *last_seconds = p->_last_seconds;
}

// show_time(s, icon) into the current bitmap
void efref_show_time(int s, int icon, uint8_t* bitmap)
{
    show_time(s, icon);
    memcpy(bitmap, _video_composite, VIDEO_COMPOSITE_HEIGHT * VIDEO_COMPOSITE_WIDTH);
}

void efref_set_last_seconds(int64_t v) { player()->_last_seconds = v; }

}  // extern "C"
