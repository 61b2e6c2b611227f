"use strict";

// Live monitor of a style transfer run.  The server sends one JSON message per iteration over /websocket
// ({_type: "STIterate", w, h, i, i_max, loss, time, gpu_ram}) and {_type: "WIDone"} at the end; /image is the
// current image as a JPEG.  At most one image request is in flight: a message that arrives meanwhile marks the
// image stale, and it is fetched again as soon as the pending load ends.

const RATE_WINDOW = 20;   // iterations in the iterations/s moving average

const el = (id) => document.getElementById(id);
const view = el("view");

let socket = null;
let finished = false;
let loading = false;
let stale = false;
let closeAfterLoad = false;
let stamps = [];          // time of the recent iterations of the current scale, in seconds

function setState(text) {
  const state = el("state");
  state.textContent = text;
  state.hidden = !text;
}

function requestImage() {
  if (loading) {
    stale = true;
    return;
  }
  loading = true;
  stale = false;
  const next = new Image();
  next.onload = () => {
    view.src = next.src;
    view.hidden = false;
    imageSettled();
  };
  next.onerror = imageSettled;   // 404 before the first image: try again with the next message
  next.src = "image?t=" + Date.now();
}

function imageSettled() {
  loading = false;
  if (stale) {
    requestImage();
  } else if (closeAfterLoad && socket) {
    socket.close();   // the final image is shown: the server need not wait for this page any longer
  }
}

function showIterate(msg) {
  el("size-w").textContent = msg.w;
  el("size-h").textContent = msg.h;
  el("iter").textContent = msg.i;
  el("iter-max").textContent = msg.i_max;
  el("loss").textContent = msg.loss.toPrecision(6);
  if (msg.i === 1) {
    stamps = [];
  }
  stamps.push(msg.time);
  if (stamps.length > RATE_WINDOW + 1) {
    stamps.shift();
  }
  if (stamps.length > 1) {
    const span = stamps[stamps.length - 1] - stamps[0];
    el("rate").textContent = span > 0 ? ((stamps.length - 1) / span).toFixed(2) : "-";
  }
  el("memory").textContent = msg.gpu_ram ? (msg.gpu_ram / 1048576).toFixed(0) + " MB" : "-";
  setState("");
}

function connect() {
  const scheme = location.protocol === "https:" ? "wss:" : "ws:";
  socket = new WebSocket(scheme + "//" + location.host + "/websocket");
  socket.onopen = () => setState("Waiting for the first iteration…");
  socket.onclose = () => {
    if (!finished) {
      setState("The connection to the server was lost.");
    }
  };
  socket.onmessage = (event) => {
    const msg = JSON.parse(event.data);
    if (msg._type === "STIterate") {
      showIterate(msg);
      requestImage();
    } else if (msg._type === "WIDone") {
      finished = true;
      closeAfterLoad = true;
      setState("Finished.");
      if (loading) {
        stale = true;   // the load in flight may predate the final image
      } else {
        requestImage();
      }
    }
  };
}

connect();
