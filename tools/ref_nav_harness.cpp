// tools/ref_nav_harness.cpp — the reference's own poster menu: ESPFlix::nav(), menu(), set_state(), load_poster(), play_pause() and
// save_pos() (espflix.cpp:704-720, 763-859, 1060-1069), compiled from the UNMODIFIED espflix.cpp, for tools/make_nav_golden.py. TEST
// INFRASTRUCTURE ONLY.
//
// As tools/ref_library_harness.cpp: espflix.cpp is included whole under `#define class struct` with every standard header first, and the
// symbols it references are stubbed. Streamer::get(url, offset) records the file asked for (a title's video file or its poster.ts) and
// the offset; Streamer::read() reports the end of the stream at once, so that load_poster()'s decode loop ends; flush_picture(mode)
// records the mode; nv_read() / nv_write() are a map of saved positions that counts its writes. loop() never returns, so the harness
// runs the branch of it a script step stands for: the pause branch (espflix.cpp:906-939) once the decoder paused with a pending action.
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

static std::string g_url;
static uint32_t g_offset = 0;
static int g_mode = -1;
static int g_writes = 0;
static std::map<std::string, int64_t> g_nv;
static std::vector<std::vector<uint8_t>> g_idx;              // every title's video.idx image
static Buffer g_buffer;

void Frame::init() {}
uint8_t* Frame::get_y(int) { return efref_composite_area; }
void Frame::erase() {}
MpegDecoder::MpegDecoder(Frame*, Frame*) {}
void MpegDecoder::flush_picture(int mode) { g_mode = mode; }
int64_t MpegDecoder::get_pts() { return g_pts; }
Buffer* MpegDecoder::pop_empty() { return &g_buffer; }
void MpegDecoder::push_full(Buffer*) {}
void MpegDecoder::reset() {}
void MpegDecoder::run() {}
int Streamer::get(const char* url, uint32_t offset, uint32_t) { g_url = url; g_offset = offset; return 0; }
void Streamer::get_rom(const uint8_t*, int) {}
static int title_of(const std::string& url)                  // ".../media/t<k>/..."
{
    const size_t at = url.find("media/t");
    return at == std::string::npos ? -1 : atoi(url.c_str() + at + 7);
}
int Streamer::get_url(const char* url, std::vector<uint8_t>& v, uint32_t offset, uint32_t len)
{
    const std::vector<uint8_t>& idx = g_idx[(size_t)title_of(url)];
    v.assign(len, 0);
    for (uint32_t i = 0; i < len && (size_t)offset + i < idx.size(); i++) v[i] = idx[offset + i];
    return (int)len;
}
ssize_t Streamer::read(uint8_t*, uint32_t, uint32_t*) { return 0; }   // the end of the stream: decode_next() returns 0
extern "C" void audio_thread(void*) {}
void beep() {}
void clear_events(int) {}
void set_events(int) {}
void wait_events(int) {}
int get_events() { return 0; }
void up_key() {}
void down_key() {}
int get_nec() { return 0; }
int64_t nv_read(const char* key) { auto it = g_nv.find(key); return it == g_nv.end() ? 0 : it->second; }
void nv_write(const char* key, int64_t pts) { g_nv[key] = pts; g_writes++; }
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

static ESPFlix* g_player = nullptr;

// loop()'s pause branch (espflix.cpp:906-939) once the decoder has paused with `pending` at get_pts() = pts
static void paused(ESPFlix* p, ESPFlix::State pending, int64_t pts)
{
    p->_pending = pending;
    p->save_pos(pending == ESPFlix::DONE ? 0 : pts, pending == ESPFlix::NAV);
    p->show_progress();
    if (p->_speed && pending != ESPFlix::DONE) {
        p->_state = ESPFlix::NAV;
        p->play_pause();
    } else if (pending == ESPFlix::NAV || pending == ESPFlix::DONE) {
        p->set_state(ESPFlix::NAV);
    } else if (pending == ESPFlix::REWIND) {
        p->rewind();
    } else if (pending == ESPFlix::FAST_FORWARD) {
        p->fast_forward();
    } else {
        video_pause(1);
        p->set_state(ESPFlix::PAUSED);
        p->_last_seconds = 0;
    }
    p->_pending = ESPFlix::NONE;
}

extern "C" {

// a service of n titles t0 .. t<n-1>, their video.idx images back to back (offsets off[n + 1]); after init_service(): NAV, nothing
// shown, no position saved
void efref_nav_load(int n, const uint8_t* idx, const uint64_t* off)
{
    if (!g_player) g_player = new ESPFlix(1);
    ESPFlix* p = g_player;
    g_idx.clear();
    p->_manifest.clear();
    p->_info.assign((size_t)n, ESPFlix::info());
    for (int i = 0; i < n; i++) {
        g_idx.emplace_back(idx + off[i], idx + off[i + 1]);
        p->_manifest.push_back("t" + std::to_string(i));
        memcpy(&p->_info[(size_t)i].idx, idx + off[i], 104);
    }
    g_nv.clear();
    p->_nav = -1;
    p->_speed = 0;
    p->_state = ESPFlix::NAV;
    p->_pending = ESPFlix::NONE;
}

// one script step (tests/nav_cases.py numbering, the library's commands): 1 PLAY = play_pause() from NAV, 6 RESUME = play_pause() from
// PAUSED; 3 / 4 FAST_FORWARD / REWIND
// and 5 PAUSE = the key while PLAYING, then the pause branch at get_pts() = pts; 8 NAV (arg = title) = nav(arg) in NAV; 9 NAV_STEP
// (arg = step) = nav(_nav + step), the left / right keys in NAV; 10 MENU = menu(), then the pause branch when it paused a PLAYING
// player; 11 DONE = the decoder ran out of bytes (_pending = DONE), then the pause branch.
void efref_nav_step(int cmd, int64_t arg, int64_t pts)
{
    ESPFlix* p = g_player;
    g_pts = pts;
    g_url.clear();
    g_offset = 0;
    g_mode = -1;
    g_writes = 0;
    switch (cmd) {
    case 1:
    case 6: p->play_pause(); break;
    case 3: paused(p, ESPFlix::FAST_FORWARD, pts); break;
    case 4: paused(p, ESPFlix::REWIND, pts); break;
    case 5: paused(p, ESPFlix::NONE, pts); break;
    case 8: p->nav((int)arg); break;
    case 9: p->nav(p->_nav + (int)arg); break;
    case 10: {
        const bool playing = p->_state == ESPFlix::PLAYING;
        p->menu();
        if (playing) paused(p, ESPFlix::NAV, pts);
        break;
    }
    case 11: paused(p, ESPFlix::DONE, pts); break;
    }
}

// what the last step did: the file asked for (0 rwd, 1 main, 2 fwd, 3 poster; -1 none) at which byte, the flush_picture() mode (-1
// none), the NVS writes, _nav, _speed, _state (1 PLAYING, 2 PAUSED, 5 NAV; -1 other), _info[_nav].pos and the saved position of every
// title (0 when none)
void efref_nav_result(int* file, uint32_t* offset, int* mode, int* writes, int* title, int* speed, int* state, int64_t* pos, int64_t* nv)
{
    ESPFlix* p = g_player;
    *file = g_url.empty() ? -1 : g_url.find("poster.ts") != std::string::npos ? 3 : g_url.find("video_rwd.ts") != std::string::npos ? 0
          : g_url.find("video_fwd.ts") != std::string::npos ? 2 : 1;
    *offset = g_offset;
    *mode = g_mode;
    *writes = g_writes;
    *title = p->_nav;
    *speed = p->_speed;
    *state = p->_state == ESPFlix::PLAYING ? 1 : p->_state == ESPFlix::PAUSED ? 2 : p->_state == ESPFlix::NAV ? 5 : -1;
    *pos = p->_nav >= 0 ? p->_info[(size_t)p->_nav].pos : 0;
    for (size_t i = 0; i < p->_manifest.size(); i++) nv[i] = nv_read(p->_manifest[i].c_str());
}

}  // extern "C"
