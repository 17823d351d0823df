// Node harness: decode an MPEG-TS file through the reference's OWN demuxer and interfaces with the
// CUDA decoder plugged in where the WASM decoder would be.  NOT RUN IN THIS REPOSITORY'S IMAGE (no
// Node); the Python twin of this script is what the tests execute (INTEGRATION.md).
//
//   node addon/decode_ts.js /path/to/jsmpeg/src clip.ts
'use strict';
const fs = require('fs');
const path = require('path');
const vm = require('vm');

const [src, clip] = process.argv.slice(2);
// the reference sources are browser scripts on a global `JSMpeg` (src/jsmpeg.js:6) and touch
// window/document at load (src/jsmpeg.js:73-77, 114-120): stub them, then load in build.sh order
global.window = {performance: require('perf_hooks').performance};
global.document = {readyState: 'loading', addEventListener() {}};
for (const f of ['jsmpeg.js', 'buffer.js', 'decoder.js', 'ts.js']) {
	vm.runInThisContext(fs.readFileSync(path.join(src, f), 'utf8'), {filename: f});
}
vm.runInThisContext(fs.readFileSync(path.join(__dirname, 'mpeg1-b200.js'), 'utf8')
	.replace("require('./jsmpeg_b200.node')", `require(${JSON.stringify(path.join(__dirname, 'build/Release/jsmpeg_b200.node'))})`),
	{filename: 'mpeg1-b200.js'});

const demuxer = new JSMpeg.Demuxer.TS({});
const video = new JSMpeg.Decoder.MPEG1VideoB200({decodeFirstFrame: false});
demuxer.connect(JSMpeg.Demuxer.TS.STREAM.VIDEO_1, video);
let pictures = 0;
video.connect({
	resize(w, h) { console.log(`sequence header: ${w}x${h}`); },
	render(y, cr, cb) { pictures++; },
});
demuxer.write(fs.readFileSync(clip).buffer);
const t0 = process.hrtime.bigint();
while (video.decode()) {}
const ms = Number(process.hrtime.bigint() - t0) / 1e6;
console.log(`${pictures} pictures in ${ms.toFixed(1)} ms`);
video.destroy();
