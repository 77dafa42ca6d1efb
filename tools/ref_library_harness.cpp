// tools/ref_library_harness.cpp — the reference's own ESPFlix navigation: play(), skip(), fast_forward(), rewind(), play_pause(),
// save_pos(), get_index() and idx_hdr::pts2offset (espflix.cpp:589-629, 787-859), compiled from the UNMODIFIED espflix.cpp, for
// tools/make_library_golden.py. TEST INFRASTRUCTURE ONLY.
//
// As tools/ref_clock_harness.cpp: espflix.cpp is included whole under `#define class struct` with every standard header first, and the
// symbols it references are stubbed. Streamer::get(url, offset) records what the player asks for, Streamer::get_url() serves the
// video.idx image the caller loaded, MpegDecoder::get_pts() returns the value the caller hands over.
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
static std::string g_url;
static uint32_t g_offset = 0, g_idx_at = 0xFFFFFFFFu;
static std::vector<uint8_t> g_idx;
int Streamer::get(const char* url, uint32_t offset, uint32_t) { g_url = url; g_offset = offset; return 0; }
void Streamer::get_rom(const uint8_t*, int) {}
int Streamer::get_url(const char*, std::vector<uint8_t>& v, uint32_t offset, uint32_t len)
{
    g_idx_at = offset;
    v.assign(len, 0);
    for (uint32_t i = 0; i < len && (size_t)offset + i < g_idx.size(); i++) v[i] = g_idx[offset + i];
    return (int)len;
}
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
        p->_manifest.assign(1, std::string("title"));
        p->_info.resize(1);
    }
    return p;
}

extern "C" {

// a title: its video.idx image; the player is on it (_nav 0) with nothing played
void efref_load(const uint8_t* idx, uint32_t bytes)
{
    ESPFlix* p = player();
    g_idx.assign(idx, idx + bytes);
    memcpy(&p->_info[0].idx, idx, 104);
    p->_nav = 0;
    p->_speed = 0;
    p->_state = ESPFlix::NAV;
}

// one command (tests/library_cases.py numbering) with get_pts() = pts. What loop() does around it: a PLAYING stream saves pos first
// (save_pos, except for PLAY_AT and RESUME); PLAY is play_pause() from NAV (the trick-mode exit, espflix.cpp:912-914); PAUSE is the
// pause branch (state PAUSED); RESUME is play_pause() from PAUSED; STOP leaves the stream stopped. cmd 8: the end of the title
// (save_pos(0), the DONE branch).
void efref_command(int cmd, int64_t arg, int64_t pts)
{
    ESPFlix* p = player();
    g_pts = pts;
    g_url.clear();
    g_idx_at = 0xFFFFFFFFu;
    if (cmd == 0) {
        p->_info[0].pos = arg;
        p->_state = ESPFlix::NAV;
        p->play_pause();
        return;
    }
    if (cmd == 8) {
        p->save_pos(0, false);
        p->_state = ESPFlix::NAV;
        return;
    }
    if (cmd != 6 && p->_state == ESPFlix::PLAYING) p->save_pos(pts, false);
    switch (cmd) {
    case 1: p->_state = ESPFlix::NAV; p->play_pause(); break;
    case 2: p->skip((int)arg); break;
    case 3: p->fast_forward(); break;
    case 4: p->rewind(); break;
    case 5: if (p->_state == ESPFlix::PLAYING) p->_state = ESPFlix::PAUSED; break;
    case 6: p->play_pause(); break;
    default: p->_state = ESPFlix::STOPPED; break;
    }
}

// what the last command did: the file asked for (0 rwd, 1 main, 2 fwd; -1 none) at which byte, the video.idx byte read (0xFFFFFFFF
// none), _speed and _info[0].pos
void efref_result(int* file, uint32_t* offset, uint32_t* idx_at, int* speed, int64_t* pos)
{
    ESPFlix* p = player();
    *file = g_url.empty() ? -1 : g_url.find("video_rwd.ts") != std::string::npos ? 0 : g_url.find("video_fwd.ts") != std::string::npos ? 2 : 1;
    *offset = g_offset;
    *idx_at = g_idx_at;
    *speed = p->_speed;
    *pos = p->_info[0].pos;
}

uint32_t efref_pts2offset(int64_t pts, int speed) { return player()->_info[0].idx.pts2offset(pts, speed); }
int64_t efref_pts2pts(int64_t pts, int speed) { return player()->_info[0].idx.pts2pts(pts, speed); }

}  // extern "C"
