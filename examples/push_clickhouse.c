/* Plain C against the C-ABI (include/tfgpu.h, include/tfgpu_sink.h): one ClickBench-shaped table's rows in row form -> tfgpu_sink_push ->
 * filter_rows + cast + ClickHouse native block + LZ4 frames on the GPU -> one INSERT over the native protocol.
 *   gcc -std=c99 -Iinclude examples/push_clickhouse.c -Ltransferia_b200 -ltfgpu -o push_clickhouse
 *   LD_LIBRARY_PATH=transferia_b200 ./push_clickhouse 127.0.0.1 9000
 * (the test suite only compiles and links it; running it needs an H100 and a ClickHouse server) */
#include <arpa/inet.h>
#include <netinet/in.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <unistd.h>

#include "tfgpu_sink.h"

static const char* SCHEMA =
    "[{\"name\":\"id\",\"type\":\"int64\",\"key\":true},{\"name\":\"url\",\"type\":\"utf8\"},{\"name\":\"ts\",\"type\":\"timestamp\"}]";
static const char* CFG =
    "{\"transformers\":[{\"filter_rows\":{\"filter\":\"id > 10\"}}],\"database\":\"default\",\"wire_fmt\":2,\"system_tables\":[\"__consumer_keeper\"]}";

/* the row image of one item: tag byte + payload per value (TF_V_*), what a shim appends while it walks ColumnValues */
static size_t put_row(unsigned char* at, long long id, const char* url, long long sec) {
    unsigned char* p = at; unsigned len = (unsigned)strlen(url), ns = 0;
    *p++ = TF_V_INT64; memcpy(p, &id, 8); p += 8;
    *p++ = TF_V_STRING; memcpy(p, &len, 4); p += 4; memcpy(p, url, len); p += len;
    *p++ = TF_V_TIME; memcpy(p, &sec, 8); p += 8; memcpy(p, &ns, 4); p += 4;
    return (size_t)(p - at);
}

static int on_event(void* ctx, const tf_sink_event* ev) {        /* control items and error rows; the row runs go to the socket */
    (void)ctx;
    printf("event type %d table %s.%s items %llu\n", ev->type, ev->out_schema, ev->out_table, (unsigned long long)ev->n_items);
    return 0;
}

int main(int argc, char** argv) {
    const char* host = argc > 1 ? argv[1] : "127.0.0.1"; int port = argc > 2 ? atoi(argv[2]) : 9000;
    tfgpu_engine* eng = NULL; tfgpu_sink* sink = NULL; tfgpu_ch_conn* ch = NULL;
    int dev = 0, rc = tfgpu_engine_create(NULL, &dev, 1, &eng);
    if (rc) { fprintf(stderr, "no engine (rc %d): there is no CPU fallback\n", rc); return 1; }
    if ((rc = tfgpu_sink_create(eng, CFG, &sink))) { fprintf(stderr, "sink rc %d\n", rc); return 1; }
    tfgpu_sink_set_callback(sink, on_event, NULL);

    int fd = socket(AF_INET, SOCK_STREAM, 0);
    struct sockaddr_in sa; memset(&sa, 0, sizeof sa); sa.sin_family = AF_INET; sa.sin_port = htons((unsigned short)port); inet_pton(AF_INET, host, &sa.sin_addr);
    if (connect(fd, (struct sockaddr*)&sa, sizeof sa) == 0 && tfgpu_ch_open(fd, "{\"database\":\"default\",\"user\":\"default\"}", &ch) == 0) {
        printf("connected: %s\n", tfgpu_ch_server_info(ch));
        tfgpu_sink_set_clickhouse(sink, ch);
    } else fprintf(stderr, "no ClickHouse at %s:%d (%s): row runs go to the callback\n", host, port, ch ? tfgpu_ch_last_error(ch) : "connect failed");

    enum { N = 1000 };
    tf_table table = {"public", "hits", SCHEMA};
    tf_item* items = calloc(N + 2, sizeof *items); unsigned char* vals = malloc((size_t)N * 128); size_t at = 0;
    items[0].kind = TF_KIND_INIT_TABLE_LOAD; items[0].old_keys_off = UINT64_MAX;
    for (int i = 0; i < N; i++) {
        tf_item* it = &items[i + 1];
        it->kind = TF_KIND_INSERT; it->n_values = 3; it->values_off = at; it->old_keys_off = UINT64_MAX; it->commit_time = 1700000000000000000ull + (unsigned)i;
        at += put_row(vals + at, i, i % 3 ? "https://example.org/a" : "", 1700000000 + i);
    }
    items[N + 1].kind = TF_KIND_DONE_TABLE_LOAD; items[N + 1].old_keys_off = UINT64_MAX;
    tf_rows rows; memset(&rows, 0, sizeof rows);
    rows.n_items = N + 2; rows.items = items; rows.n_tables = 1; rows.tables = &table; rows.values = vals; rows.values_len = at;

    rc = tfgpu_sink_push(sink, &rows);                              /* Sinker.Push: > 0 retriable, < 0 fatal */
    tf_sink_stats st; tfgpu_sink_stats(sink, &st);
    printf("push rc %d (%s): %llu change items, %llu row events, %llu wire bytes\n", rc, rc ? tfgpu_sink_last_error(sink) : "ok",
           (unsigned long long)st.change_items_pushed, (unsigned long long)st.row_events_pushed, (unsigned long long)st.wire_bytes);

    if (ch) tfgpu_ch_close(ch);
    close(fd); tfgpu_sink_destroy(sink); tfgpu_engine_destroy(eng); free(items); free(vals);
    return rc != 0;
}
